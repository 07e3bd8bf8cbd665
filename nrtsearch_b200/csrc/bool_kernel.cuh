// Batched BooleanQuery execution over HBM-resident postings: window engine + slice merge.
//
// Replaces, for a whole batch of queries at once, the per-query chain
//   IndexSearcher.search -> BooleanWeight.bulkScorer -> (MaxScoreBulkScorer | ConjunctionDISI) ->
//   TermScorer/BM25Scorer -> TopScoreDocCollector
// that the reference drives from src/main/java/com/yelp/nrtsearch/server/handler/SearchHandler.java:1412.
//
// Work item = (doc slice, query). A CTA sweeps its slice in windows of W docs:
//   pass 1 (scatter): every posting of every term clause in the window stores its saturated tf byte
//                     into byte `slot` of a W-entry shared-memory word array (no atomics: doc ids
//                     are unique inside one posting list and the passes are barrier separated);
//   pass 2 (emit):    the postings of the DRIVER clauses are re-read; the lowest driver clause present
//                     in a doc's word "owns" the doc, clears the word, evaluates the boolean
//                     constraints, scores the matched clauses with Lucene's BM25 float formula, sums
//                     in double in clause order, and offers (score, doc) to the CTA's candidate
//                     buffer if it beats the query's running threshold theta;
//   pass 3 (clean):   non-driver clauses clear the words pass 2 did not visit.
// Smem cost is proportional to postings, not to W. theta is a 64-bit (score, ~doc) key shared by all
// slices of a query through one global atomicMax word -- the device analogue of the reference's
// LazyMaxScoreAccumulator (src/main/java/org/apache/lucene/search/LazyMaxScoreAccumulator.java:21-70),
// used here only to drop hits that provably cannot enter the top-k (results stay exact).
// Query trees (tree batches, bool_window_kernel<true, *>) change pass 2 only: the drivers are the term leaves of the root's
// cover (batch_plan.inc compile_tree), and a doc is evaluated node by node (eval_node) instead of by one clause list.
// Additional collectors (nrtgpu_search_tree_aggs, bool_window_kernel<kTree, true>): every matching doc is also handed to
// agg_collect with its score, where pass 2 counts it, as the probe kernel's generic instantiation does.
// Multi-phrase unions (tree batches whose term slots include call unions, bool_window_union_kernel): a union slot's list is
// the call's union entries (union_kernel.cuh) instead of the image's postings, a presence byte in pass 1; the phrase
// matcher reads its merged positions and a scoring one-position slot its entry's score (query_eval.cuh SmemUnions). A
// block join's (parent, score) entries (join_kernel.cuh) are read the same way.
// Child pass of block joins (bool_window_emit_kernel): the tree, union-capable body with kEmit, run over the joins' child
// queries; every match is appended to the call's join keys instead of offered to a top-k, with no theta, no slice lists,
// no totalHits and no deadline (it runs when the batch is built, as the union build does).
#pragma once
#include <type_traits>
#include "query_eval.cuh"
#include "collect_kernel.cuh"
#include "union_kernel.cuh"

namespace nrtgpu {

// (DevClause, DevQuery, the clause / slot / top_k limits and the window size: batch_plan.h)
constexpr int kCandCap = 4096;      // candidate buffer (keys) per CTA, power of two
constexpr int kThreads = 512;

struct BoolLaunch {
  DevIndexView ix;
  const DevClause* clauses;
  const DevQuery* queries;
  const int32_t* work_query;   // [n_work] query index per work item (slice-major order)
  const int32_t* work_slice;   // [n_work]
  int32_t n_work;
  int32_t n_slices;
  int32_t top_k;
  uint64_t* theta;             // [nq] running k-th best key (0 = none yet)
  unsigned long long* total_hits;  // [nq]
  uint64_t* slice_keys;        // [nq][n_slices][top_k]
  int32_t* slice_cnt;          // [nq][n_slices]
  // deadline, checked when a work item starts (deadline_passed, as in the probe kernel): a late item writes no keys,
  // counts no hits and flags its query
  long long deadline_ns;       // 0: no deadline; < 0: already expired
  unsigned long long* clock0;
  int32_t* timed_out;          // [nq]
  // tree batches (batch_plan.h DevNode): the nodes of query q are nodes[node_begin[q], node_begin[q + 1])
  const DevNode* nodes;
  const int32_t* node_begin;
  // tree batches with phrases (batch_plan.h DevPhrase): the records of query q are phrases[phrase_begin[q], phrase_begin[q + 1])
  const DevPhrase* phrases;
  const int32_t* phrase_begin;
  // additional collectors (the kAggs instantiations; device pointer)
  const AggLaunch* aggs;
};

template <bool kTree>
struct BoolSmemT {
  uint64_t slots[kWindowDocs];   // one tf byte per term slot
  uint64_t cand[kCandCap];
  uint32_t bounds[kMaxTermSlots][kSliceWindows + 1];
  float cache[kMaxTermSlots][256];
  DevClause cl[kTree ? kMaxTreeClauses : kMaxClauses];
  DevQuery q;
  int cand_count;
  int skip;   // the work item started after the deadline
  unsigned long long theta;
};
using BoolSmem = BoolSmemT<false>;
// tree batches: the query's nodes next to its clauses
struct BoolTreeSmem : BoolSmemT<true> {
  DevNode nodes[kMaxTreeNodes];
  DevPhrase phrases[kMaxTreePhrases];
  int n_nodes;
  int n_phrases;
};
// tree batches with multi-phrase unions: the call's union entries
struct BoolLaunchU : BoolLaunch {
  UnionView u;
};
struct BoolTreeSmemU : BoolTreeSmem {
  UnionView u;
};
template <> struct SmemUnions<BoolTreeSmemU> : std::true_type {};
// the child pass of block joins: where its matches go (query q is join q - join_q0's child query)
struct BoolLaunchJ : BoolLaunchU {
  uint64_t* emit_keys;          // [emit_cap] (join << 32 | child doc)
  float* emit_scores;           // [emit_cap]
  unsigned int* emit_count;
  int64_t emit_cap;
  int32_t join_q0;
};

// the list of a term slot: the image's postings, or (kUnion) the call's union entries
template <bool kUnion, class Launch>
__device__ __forceinline__ const int32_t* list_docs(const Launch& L, const DevClause& c) {
  if constexpr (kUnion) {
    if (c.plane == kUnionList) return L.u.docs + c.post_base;
  }
  return L.ix.post_docs + c.post_base;
}

// the clauses of sm.q on one candidate doc; slot holds the doc's tf byte of every term slot
__device__ __forceinline__ bool evaluate_doc(const DevIndexView& ix, const BoolSmem& sm, int32_t doc,
                                             uint64_t slot, float* out_score) {
  auto term = [&](const DevClause& c, float* s) {
    const uint32_t b = (uint32_t)((slot >> (8 * c.slot)) & 0xff);
    if (b == 0) return false;
    if (c.scoring) {
      const float f = (b == 255u) ? exact_freq_slow(ix, c, doc) : (float)b;
      const uint8_t* nrm = ix.norms[c.field];
      const uint32_t nb = nrm ? (uint32_t)nrm[doc] : 1u;
      *s = bm25_score(c.weight, f, sm.cache[c.slot][nb]);
    }
    return true;
  };
  return eval_clauses(ix, sm.q, sm.cl, doc, presence_mask(slot), term, out_score);
}

// a phrase term's posting in the window engine: a lower_bound inside its slot's bounds of the doc's window (sm.bounds)
__device__ __forceinline__ uint32_t phrase_posting(const DevIndexView& ix, const BoolTreeSmem& sm, const DevClause& t, int32_t doc) {
  const int w = (doc & (kWideSliceDocs - 1)) / kWindowDocs;   // the doc's window in its slice
  const int32_t* docs = ix.post_docs + t.post_base;
  uint32_t lo = sm.bounds[t.slot][w], hi = sm.bounds[t.slot][w + 1];
  while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (__ldg(docs + m) < doc) lo = m + 1; else hi = m; }
  return lo;
}

// ... of a slot that may be a union
__device__ __forceinline__ uint32_t phrase_posting(const DevIndexView& ix, const BoolTreeSmemU& sm, const DevClause& t, int32_t doc) {
  const int w = (doc & (kWideSliceDocs - 1)) / kWindowDocs;
  const int32_t* docs = (t.plane == kUnionList ? sm.u.docs : ix.post_docs) + t.post_base;
  uint32_t lo = sm.bounds[t.slot][w], hi = sm.bounds[t.slot][w + 1];
  while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (__ldg(docs + m) < doc) lo = m + 1; else hi = m; }
  return lo;
}

// the query tree of sm on one candidate doc
__device__ __forceinline__ bool evaluate_doc(const DevIndexView& ix, const BoolTreeSmem& sm, int32_t doc, uint64_t slot,
                                             float* out_score) {
  return eval_tree(ix, sm, doc, slot, out_score);
}
__device__ __forceinline__ bool evaluate_doc(const DevIndexView& ix, const BoolTreeSmemU& sm, int32_t doc, uint64_t slot,
                                             float* out_score) {
  return eval_tree(ix, sm, doc, slot, out_score);
}

// kTree: a tree batch (sm holds the query's nodes, evaluate_doc walks them); otherwise flat BooleanQuerys.
// kAggs: every matching doc also goes to the collectors of L.aggs (the other instantiations never read it); kMulti: they
// count a SORTED_SET keyword column (agg_collect<true>); kUnion (tree batches): term slots may be call unions (L.u);
// kEmit (the child pass of block joins, BoolLaunchJ): every match is appended to L.emit_* instead
template <bool kTree, bool kAggs, bool kMulti, bool kUnion, class Launch, bool kEmit = false>
__device__ __forceinline__ void bool_window_body(const Launch& L, unsigned char* smem_raw) {
  using Smem = typename std::conditional<kUnion, BoolTreeSmemU, typename std::conditional<kTree, BoolTreeSmem, BoolSmem>::type>::type;
  Smem& sm = *reinterpret_cast<Smem*>(smem_raw);
  const int tid = threadIdx.x;
  const int lane = tid & 31;

  for (int wi = blockIdx.x; wi < L.n_work; wi += gridDim.x) {
    const int qi = L.work_query[wi];
    const int slice = L.work_slice[wi];
    __syncthreads();  // previous work item fully retired
    if (tid == 0) {
      sm.q = L.queries[qi];
      sm.cand_count = 0;
      if constexpr (kEmit) {
        sm.theta = 0ull; sm.skip = 0;
      } else {
        sm.theta = *(volatile unsigned long long*)&L.theta[qi];
        sm.skip = L.deadline_ns && deadline_passed(L.deadline_ns, L.clock0);
        if (sm.skip) L.timed_out[qi] = 1;
      }
      if constexpr (kTree) {
        sm.n_nodes = L.node_begin[qi + 1] - L.node_begin[qi];
        sm.n_phrases = L.phrase_begin ? L.phrase_begin[qi + 1] - L.phrase_begin[qi] : 0;
      }
      if constexpr (kUnion) sm.u = L.u;
    }
    __syncthreads();
    if (sm.skip) continue;   // (CTA-uniform) slice_cnt stays 0: the slice contributes no keys
    const int ncl = sm.q.n_clauses;
    if (tid < ncl) sm.cl[tid] = L.clauses[sm.q.clause_begin + tid];
    if constexpr (kTree) {
      if (tid < sm.n_nodes) sm.nodes[tid] = L.nodes[L.node_begin[qi] + tid];
      if (tid < sm.n_phrases) sm.phrases[tid] = L.phrases[L.phrase_begin[qi] + tid];
    }
    for (int i = tid; i < kWindowDocs; i += kThreads) sm.slots[i] = 0;
    __syncthreads();
    // per-slot BM25 caches
    for (int i = tid; i < ncl * 256; i += kThreads) {
      int c = i >> 8;
      if (sm.cl[c].kind == NRTGPU_TERM) sm.cache[sm.cl[c].slot][i & 255] = L.ix.caches[sm.cl[c].field * 256 + (i & 255)];
    }
    const int32_t slice_base = slice * kWideSliceDocs;
    int32_t slice_end = slice_base + kWideSliceDocs;
    if (slice_end > L.ix.n_docs || slice_end < 0) slice_end = L.ix.n_docs;
    const int nwin = (slice_end - slice_base + kWindowDocs - 1) / kWindowDocs;
    // posting bounds of every term clause at every window boundary (lower_bound over the full list)
    for (int i = tid; i < ncl * (kSliceWindows + 1); i += kThreads) {
      int c = i / (kSliceWindows + 1), w = i % (kSliceWindows + 1);
      if (sm.cl[c].kind != NRTGPU_TERM) continue;
      int64_t target64 = (int64_t)slice_base + (int64_t)w * kWindowDocs;
      int32_t target = target64 > (int64_t)slice_end ? slice_end : (int32_t)target64;
      const int32_t* docs = list_docs<kUnion>(L, sm.cl[c]);
      int lo = 0, hi = sm.cl[c].n_post;
      while (lo < hi) { int mid = (lo + hi) >> 1; if (__ldg(docs + mid) < target) lo = mid + 1; else hi = mid; }
      sm.bounds[sm.cl[c].slot][w] = (uint32_t)lo;
    }
    __syncthreads();

    unsigned long long my_hits = 0;
    int cand_ub = 0;  // CTA-uniform upper bound of cand_count
    const bool dense = sm.q.dense_driver != 0;
    const bool has_after = sm.q.has_after != 0;
    const uint64_t after_key = sm.q.after_key;

    for (int w = 0; w < nwin; ++w) {
      const int32_t wbase = slice_base + w * kWindowDocs;
      const int32_t wlen = min(kWindowDocs, slice_end - wbase);
      // ---------------- pass 1: scatter tf bytes
      bool any = dense;
      for (int c = 0; c < ncl; ++c) {
        if (sm.cl[c].kind != NRTGPU_TERM) continue;
        const int s = sm.cl[c].slot;
        const uint32_t b0 = sm.bounds[s][w], b1 = sm.bounds[s][w + 1];
        if (b1 > b0) any = true;
        const int32_t* docs = list_docs<kUnion>(L, sm.cl[c]);
        const uint8_t* f8 = L.ix.post_f8 + sm.cl[c].post_base;
        bool scoring = sm.cl[c].scoring != 0;
        if constexpr (kUnion) scoring = scoring && sm.cl[c].plane != kUnionList;   // a union slot: a presence byte
        unsigned char* slot_bytes = reinterpret_cast<unsigned char*>(sm.slots);
        for (uint32_t p = b0 + tid; p < b1; p += kThreads) {
          int32_t d = docs[p] - wbase;
          unsigned char f = scoring ? f8[p] : (unsigned char)1;
          slot_bytes[(size_t)d * sizeof(uint64_t) + s] = f;
        }
      }
      if (!any) continue;  // CTA-uniform: no postings in this window
      __syncthreads();
      // ---------------- pass 2: emit
      auto offer = [&](bool matched, int32_t doc, float score) {
        // converged call (all lanes of the warp)
        if constexpr (kEmit) {   // a warp-aggregated append of the warp's matches
          const unsigned bal = __ballot_sync(0xffffffffu, matched);
          if (bal) {
            unsigned int base = 0;
            if (lane == 0) base = atomicAdd(L.emit_count, (unsigned int)__popc(bal));
            base = __shfl_sync(0xffffffffu, base, 0);
            const int64_t at = (int64_t)base + __popc(bal & ((1u << lane) - 1));
            if (matched && at < L.emit_cap) {
              L.emit_keys[at] = ((uint64_t)(uint32_t)(qi - L.join_q0) << 32) | (uint32_t)doc;
              L.emit_scores[at] = score;
            }
          }
          return;
        }
        bool is_cand = false;
        uint64_t key = 0;
        if (matched) {
          ++my_hits;
          if constexpr (kAggs) agg_collect<kMulti>(*L.aggs, L.ix, qi, doc, score);   // additional collectors see every matching doc
          key = make_key(score, doc);
          is_cand = key > sm.theta && (!has_after || key < after_key);
        }
        unsigned bal = __ballot_sync(0xffffffffu, is_cand);
        if (bal) {
          int base = 0;
          if (lane == 0) base = atomicAdd(&sm.cand_count, __popc(bal));
          base = __shfl_sync(0xffffffffu, base, 0);
          if (is_cand) sm.cand[base + __popc(bal & ((1u << lane) - 1))] = key;
        }
      };
      auto round_end = [&]() {
        if constexpr (kEmit) return;
        cand_ub += kThreads;
        if (cand_ub > kCandCap - kThreads) {
          __syncthreads();
          int n = sm.cand_count;
          if (n > kCandCap - kThreads) { flush_top_k(sm.cand, sm.cand_count, kCandCap, L.top_k, 0ull, &L.theta[qi], sm.theta); n = sm.cand_count; }
          cand_ub = n;
        }
      };
      if (!dense) {
        for (int c = 0; c < ncl; ++c) {
          if (sm.cl[c].kind != NRTGPU_TERM) continue;
          const int s = sm.cl[c].slot;
          if (!((sm.q.driver_mask >> s) & 1u)) continue;
          // bytes of lower driver slots
          uint64_t below = 0;
          for (int j = 0; j < s; ++j) if ((sm.q.driver_mask >> j) & 1u) below |= (uint64_t)0xff << (8 * j);
          const uint64_t own = (uint64_t)0xff << (8 * s);
          const uint32_t b0 = sm.bounds[s][w], b1 = sm.bounds[s][w + 1];
          const int32_t* docs = list_docs<kUnion>(L, sm.cl[c]);
          for (uint32_t p0 = b0; p0 < b1; p0 += kThreads) {
            uint32_t p = p0 + tid;
            bool matched = false; int32_t doc = 0; float score = 0.0f;
            if (p < b1) {
              doc = docs[p];
              uint64_t v = sm.slots[doc - wbase];
              if ((v & below) == 0 && (v & own) != 0) {
                sm.slots[doc - wbase] = 0;
                matched = evaluate_doc(L.ix, sm, doc, v, &score);
              }
            }
            offer(matched, doc, score);
            round_end();
          }
          __syncthreads();   // the words this list cleared are seen cleared by the next driver list (either order gave the same
                             // result -- the doc is skipped -- but the ordering is now explicit: racecheck-clean)
        }
      } else {
        for (int i0 = 0; i0 < wlen; i0 += kThreads) {
          int i = i0 + tid;
          bool matched = false; int32_t doc = wbase + i; float score = 0.0f;
          if (i < wlen) {
            uint64_t v = sm.slots[i];
            if (v) sm.slots[i] = 0;
            matched = evaluate_doc(L.ix, sm, doc, v, &score);
          }
          offer(matched, doc, score);
          round_end();
        }
      }
      __syncthreads();
      // ---------------- pass 3: clear words of non-driver clauses
      if (!dense && sm.q.has_non_driver) {
        for (int c = 0; c < ncl; ++c) {
          if (sm.cl[c].kind != NRTGPU_TERM) continue;
          const int s = sm.cl[c].slot;
          if ((sm.q.driver_mask >> s) & 1u) continue;
          const uint32_t b0 = sm.bounds[s][w], b1 = sm.bounds[s][w + 1];
          const int32_t* docs = list_docs<kUnion>(L, sm.cl[c]);
          for (uint32_t p = b0 + tid; p < b1; p += kThreads) sm.slots[docs[p] - wbase] = 0;
        }
        __syncthreads();
      }
    }
    // ---------------- finish the work item
    if constexpr (kEmit) continue;
    flush_top_k(sm.cand, sm.cand_count, kCandCap, L.top_k, 0ull, &L.theta[qi], sm.theta);
    const int keep = sm.cand_count;
    uint64_t* out = L.slice_keys + ((size_t)qi * L.n_slices + slice) * L.top_k;
    for (int i = tid; i < keep; i += kThreads) out[i] = sm.cand[i];
    if (tid == 0) L.slice_cnt[(size_t)qi * L.n_slices + slice] = keep;
    // total hits
    for (int o = 16; o > 0; o >>= 1) my_hits += __shfl_xor_sync(0xffffffffu, my_hits, o);
    if (lane == 0 && my_hits) atomicAdd(&L.total_hits[qi], my_hits);
  }
}

template <bool kTree, bool kAggs, bool kMulti = false>
__global__ void __launch_bounds__(kThreads, 2) bool_window_kernel(const __grid_constant__ BoolLaunch L) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  bool_window_body<kTree, kAggs, kMulti, false>(L, smem_raw);
}

// tree batches with multi-phrase unions (shared memory: sizeof(BoolTreeSmemU))
template <bool kAggs, bool kMulti = false>
__global__ void __launch_bounds__(kThreads, 2) bool_window_union_kernel(const __grid_constant__ BoolLaunchU L) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  bool_window_body<true, kAggs, kMulti, true>(L, smem_raw);
}

// the child pass of block joins (shared memory: sizeof(BoolTreeSmemU))
__global__ void __launch_bounds__(kThreads, 2) bool_window_emit_kernel(const __grid_constant__ BoolLaunchJ L) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  bool_window_body<true, false, false, true, BoolLaunchJ, true>(L, smem_raw);
}

// ---- per-query merge of the slice lists (TopDocs.merge semantics: key order is total) ----
struct MergeLaunch {
  const uint64_t* slice_keys;  // [nq][n_lists][top_k]
  const int32_t* slice_cnt;    // [nq][n_lists]
  int32_t n_lists, top_k, nq;
  int32_t doc_base;
  int32_t* out_docs; float* out_scores; int32_t* out_counts;
  // optional: per-query totalHits / relation of the shard written next to the hits (the packed record of the one
  // all-gather of a multi-GPU step, nrtgpu_batch_bind_packed)
  const unsigned long long* total_hits; const int32_t* pruned; int32_t* terminated;
  long long terminate_after;                  // > 0: a query with more hits than this terminated early (TerminateAfterWrapper.java:150-158)
  long long* out_total; int32_t* out_flags;   // flags: bit 0 relation GREATER_THAN_OR_EQUAL_TO, bit 1 terminated early
  const unsigned long long* known_hits = nullptr;   // optional [nq]: docs known to match (reported totalHits = max(counted, known))
  const uint64_t* theta = nullptr;            // optional [nq]: the k-th best key some work item published (>= top_k keys are >= it):
                                              // smaller keys cannot be in the merged page and are dropped before the sort
};

constexpr int kMergeThreads = 256;
constexpr int kMergeCap = 4096;

__global__ void __launch_bounds__(kMergeThreads) merge_slices_kernel(MergeLaunch M) {
  __shared__ uint64_t keys[kMergeCap];
  __shared__ int32_t s_cnt[kMergeThreads];
  __shared__ int32_t s_nz[kMergeThreads];   // the non-empty lists of a chunk of list counts
  __shared__ int32_t s_off[kMergeThreads];
  __shared__ int32_t s_nnz;
  __shared__ int32_t s_fill;
  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  const uint64_t floor_key = M.theta ? M.theta[q] : 0ull;
  int have = 0;        // keys[0..have) hold the best so far
  bool dirty = false;  // ... unsorted / not yet cut to top_k
  auto sort_and_cut = [&]() {
    const int m = next_pow2(have < 2 ? 2 : have);
    __syncthreads();
    for (int i = have + tid; i < m; i += kMergeThreads) keys[i] = 0ull;
    __syncthreads();
    block_bitonic_sort_desc(keys, m);
    have = have < M.top_k ? have : M.top_k;
    dirty = false;
    __syncthreads();
  };
  // the list counts are read kMergeThreads at a time (most lists of a query whose work items were not split are empty);
  // non-empty lists are appended while they fit, the buffer sorted and cut to top_k when the next one does not
  for (int l0 = 0; l0 < M.n_lists; l0 += kMergeThreads) {
    __syncthreads();
    if (tid == 0) s_nnz = 0;
    __syncthreads();
    const int l = l0 + tid;
    const int c = l < M.n_lists ? M.slice_cnt[(size_t)q * M.n_lists + l] : 0;
    if (c > 0) { const int p = atomicAdd(&s_nnz, 1); s_nz[p] = l; s_cnt[p] = c; }
    __syncthreads();
    const int nnz = s_nnz;
    // exclusive prefix of the non-empty lists' counts (block-wide Hillis-Steele scan): the keys of the chunk become one flat
    // range that the 256 threads read with independent loads, instead of list after list
    s_off[tid] = tid < nnz ? s_cnt[tid] : 0;
    __syncthreads();
    for (int d = 1; d < kMergeThreads; d <<= 1) {
      const int v = tid >= d ? s_off[tid - d] : 0;
      __syncthreads();
      s_off[tid] += v;
      __syncthreads();
    }
    // (inclusive scan: s_off[i] = keys of lists 0..i of the chunk)
    int i0 = 0;
    while (i0 < nnz) {
      // the longest run of lists [i0, i1) that fits behind the keys kept so far (worst case: no key below the floor)
      const int base = i0 ? s_off[i0 - 1] : 0;
      if (have + (s_off[i0] - base) > kMergeCap) sort_and_cut();   // room for list i0 at least (after the cut: <= top_k + top_k keys)
      int i1 = i0 + 1;
      while (i1 < nnz && have + (s_off[i1] - base) <= kMergeCap) ++i1;
      const int n_flat = s_off[i1 - 1] - base;
      __syncthreads();
      if (tid == 0) s_fill = have;
      __syncthreads();
      for (int e0 = tid; e0 < n_flat; e0 += 4 * kMergeThreads) {   // four independent loads in flight per thread
        uint64_t kk[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int e = e0 + u * kMergeThreads;
          kk[u] = 0ull;
          if (e < n_flat) {
            int lo = i0, hi = i1;   // list of flat element e: the first i in [i0, i1) with s_off[i] - base > e
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_off[mid] - base > e) hi = mid; else lo = mid + 1; }
            kk[u] = M.slice_keys[((size_t)q * M.n_lists + s_nz[lo]) * M.top_k + (e - (lo > i0 ? s_off[lo - 1] - base : 0))];
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (kk[u] != 0ull && kk[u] >= floor_key) keys[atomicAdd(&s_fill, 1)] = kk[u];   // (a real key is never 0)
      }
      __syncthreads();
      if (s_fill > have) dirty = true;
      have = s_fill;
      i0 = i1;
    }
  }
  if (dirty) sort_and_cut();
  if (M.n_lists <= 0) have = 0;
  __syncthreads();
  for (int i = tid; i < M.top_k; i += kMergeThreads) {   // slots past the count: doc 0, score 0.0 (include/nrtgpu.h)
    const uint64_t k = keys[i < have ? i : 0];
    M.out_docs[(size_t)q * M.top_k + i] = i < have ? key_doc(k) + M.doc_base : 0;
    M.out_scores[(size_t)q * M.top_k + i] = i < have ? key_score(k) : 0.0f;
  }
  if (tid == 0) {
    M.out_counts[q] = have;
    if (M.terminate_after > 0 && M.terminated && M.total_hits && (long long)M.total_hits[q] > M.terminate_after) M.terminated[q] = 1;
    const bool term = M.terminated && M.terminated[q];
    if (M.out_total) {
      long long t = M.total_hits ? (long long)M.total_hits[q] : 0ll;
      if (M.known_hits && M.pruned && M.pruned[q] && (long long)M.known_hits[q] > t) t = (long long)M.known_hits[q];   // a lower bound either way
      M.out_total[q] = t;
    }
    if (M.out_flags) M.out_flags[q] = ((M.pruned && M.pruned[q]) || term ? 1 : 0) | (term ? 2 : 0);
  }
}

// TopDocs.merge over lists of (doc, score) pairs (cross-shard merge after the NCCL all-gather).
struct MergePairsLaunch {
  const int32_t* docs; const float* scores; const int32_t* counts;  // list l: docs + l * stride_hits [nq][top_k], counts + l * stride_counts [nq]
  int64_t stride_hits, stride_counts;   // elements between consecutive lists
  int32_t n_lists, top_k, nq;
  int32_t* out_docs; float* out_scores; int32_t* out_counts;
  // optional (packed records): totalHits summed, flags ORed over the shards (TopDocs.merge: relation GTE if any input is)
  const long long* totals; const int32_t* flags; int64_t stride_totals, stride_flags;
  long long* out_total; int32_t* out_flags;
};

__global__ void __launch_bounds__(kMergeThreads) merge_pairs_kernel(MergePairsLaunch M) {
  __shared__ uint64_t keys[kMergeCap];
  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  int have = 0;
  int l = 0;
  while (l < M.n_lists) {
    int fill = have;
    int l_end = l;
    __syncthreads();
    while (l_end < M.n_lists) {
      int c = M.counts[(size_t)l_end * M.stride_counts + q];
      if (fill + c > kMergeCap) break;
      size_t base = (size_t)l_end * M.stride_hits + (size_t)q * M.top_k;
      for (int i = tid; i < c; i += kMergeThreads) keys[fill + i] = make_key(M.scores[base + i], M.docs[base + i]);
      fill += c; ++l_end;
    }
    l = l_end;
    int m = next_pow2(fill < 2 ? 2 : fill);
    for (int i = fill + tid; i < m; i += kMergeThreads) keys[i] = 0ull;
    __syncthreads();
    block_bitonic_sort_desc(keys, m);
    have = fill < M.top_k ? fill : M.top_k;
  }
  __syncthreads();
  for (int i = tid; i < M.top_k; i += kMergeThreads) {   // slots past the count: doc 0, score 0.0 (include/nrtgpu.h)
    const uint64_t k = keys[i < have ? i : 0];
    M.out_docs[(size_t)q * M.top_k + i] = i < have ? key_doc(k) : 0;
    M.out_scores[(size_t)q * M.top_k + i] = i < have ? key_score(k) : 0.0f;
  }
  if (tid == 0) {
    M.out_counts[q] = have;
    if (M.out_total) {
      long long t = 0; int32_t f = 0;
      for (int l2 = 0; l2 < M.n_lists; ++l2) { t += M.totals[(size_t)l2 * M.stride_totals + q]; f |= M.flags[(size_t)l2 * M.stride_flags + q]; }
      M.out_total[q] = t; M.out_flags[q] = f;
    }
  }
}

}  // namespace nrtgpu
