// Kernels either side of the top-k: the second pass of QueryRescorer (a query evaluated on a given hit list), the
// fetch phase on doc-value columns, and the aggregating "additional collectors" (terms / min / max / sum).
//   reference: src/main/java/com/yelp/nrtsearch/server/rescore/QueryRescore.java:39-57 (Lucene QueryRescorer.rescore),
//              .../handler/SearchHandler.java:397-522 (fetch: FillDocsTask / LoadedDocValues),
//              .../search/collectors/additional/{Int,Long,Float,Double}TermsCollectorManager.java, Max/Min/SumCollectorManager.java,
//              fan-out at .../search/SearchCollectorManager.java:192-198.
#pragma once
#include <cfloat>
#include "query_eval.cuh"
#include "../../include/nrtgpu.h"

namespace nrtgpu {

// exact tf of (term clause, doc): dense byte plane when the term has one, else a binary search of its postings
__device__ __forceinline__ float term_freq_of(const DevIndexView& ix, const DevClause& c, int32_t doc, bool* present) {
  if (c.plane >= 0 && ix.dense_tf) {
    const uint32_t b = ix.dense_tf[(size_t)c.plane * (size_t)ix.dense_stride + doc];
    *present = b != 0;
    if (b != 255u) return (float)b;
    return exact_freq_slow(ix, c, doc);
  }
  const int32_t* docs = ix.post_docs + c.post_base;
  int lo = 0, hi = c.n_post;
  while (lo < hi) { const int m = (lo + hi) >> 1; if (__ldg(docs + m) < doc) lo = m + 1; else hi = m; }
  *present = lo < c.n_post && __ldg(docs + lo) == doc;
  if (!*present) return 0.0f;
  const uint32_t b = ix.post_f8[c.post_base + lo];
  if (b != 255u) return (float)b;
  return exact_freq_slow(ix, c, doc);
}

// query q on one doc of the leaf; term presence is found clause by clause, so no presence mask is known up front
__device__ __forceinline__ bool eval_query_on_doc(const DevIndexView& ix, const DevQuery& q, const DevClause* __restrict__ cl,
                                                  int32_t doc, float* out_score) {
  if (q.empty) return false;
  auto term = [&](const DevClause& c, float* s) {
    bool present;
    const float f = term_freq_of(ix, c, doc, &present);
    if (present && c.scoring) {
      const uint8_t* nrm = ix.norms[c.field];
      const uint32_t nb = nrm ? (uint32_t)nrm[doc] : 1u;
      *s = bm25_score(c.weight, f, ix.caches[c.field * 256 + nb]);
    }
    return present;
  };
  return eval_clauses(ix, q, cl, doc, q.req_term_mask, term, out_score);
}

// QueryRescorer second pass: query q on its own first-pass hits
struct ScoreDocsLaunch {
  DevIndexView ix;
  const DevClause* clauses; const DevQuery* queries;
  int32_t nq, n_hits;
  const int32_t* docs;     // [nq][n_hits] global doc ids
  const int32_t* counts;   // [nq] or NULL
  uint8_t* out_matches; float* out_scores;
};

__global__ void score_docs_kernel(const __grid_constant__ ScoreDocsLaunch L) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L.nq * L.n_hits) return;
  const int q = i / L.n_hits, r = i % L.n_hits;
  uint8_t m = 0; float s = 0.0f;
  if (r < (L.counts ? L.counts[q] : L.n_hits)) {
    const int64_t local = (int64_t)L.docs[i] - L.ix.doc_base;
    if (local >= 0 && local < L.ix.n_docs) {
      const DevQuery dq = L.queries[q];
      float sc;
      if (eval_query_on_doc(L.ix, dq, L.clauses + dq.clause_begin, (int32_t)local, &sc)) { m = 1; s = sc; }
    }
  }
  L.out_matches[i] = m; L.out_scores[i] = s;
}

// QueryRescorer second pass of a tree batch (query trees, phrase leaves): one CTA per (query, chunk of kScoreTreeThreads
// hits), the query's clauses, nodes, phrase records and per-slot BM25 caches staged once per CTA, one hit per thread
struct ScoreDocsTreeLaunch : ScoreDocsLaunch {
  const DevNode* nodes; const int32_t* node_begin;        // the nodes of query q: nodes[node_begin[q], node_begin[q + 1])
  const DevPhrase* phrases; const int32_t* phrase_begin;  // its phrase records: phrases[phrase_begin[q], phrase_begin[q + 1])
  int32_t n_chunks;                                       // CTAs per query: blockIdx.x = q * n_chunks + chunk
};

constexpr int kScoreTreeThreads = 256;

struct ScoreTreeSmem {
  DevClause cl[kMaxTreeClauses];
  DevNode nodes[kMaxTreeNodes];
  DevPhrase phrases[kMaxTreePhrases];
  float cache[kMaxTermSlots][256];
  uint32_t post[kMaxTermSlots][kScoreTreeThreads];   // the posting (index in its term's list) of each slot present in a thread's doc
  DevQuery q;
  int n_nodes;
};

// a phrase term's posting in the second pass: the one the slot lookup found
__device__ __forceinline__ uint32_t phrase_posting(const DevIndexView&, const ScoreTreeSmem& sm, const DevClause& t, int32_t) {
  return sm.post[t.slot][threadIdx.x];
}

// The tf byte and posting of term clause c in doc: a lower_bound over the term's postings, narrowed by its granule row (the
// index-time skip data) to the postings of the doc's 1024-doc granule when it has one. 0: the doc holds no posting.
__device__ __forceinline__ uint32_t slot_lookup(const DevIndexView& ix, const DevClause& c, int32_t doc, uint32_t* post) {
  const int32_t* docs = ix.post_docs + c.post_base;
  uint32_t lo = 0, hi = (uint32_t)c.n_post;
  if (c.gran_row >= 0) {
    const uint32_t* row = ix.gran_tab + (size_t)c.gran_row * (size_t)(ix.n_gran + 1) + (doc >> v3::kLogGran);
    lo = __ldg(row); hi = __ldg(row + 1);
  }
  const uint32_t end = hi;
  while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (__ldg(docs + m) < doc) lo = m + 1; else hi = m; }
  if (lo == end || __ldg(docs + lo) != doc) return 0u;
  *post = lo;
  return c.scoring ? (uint32_t)__ldg(ix.post_f8 + c.post_base + lo) : 1u;   // (pass 1 of the window engine stores the same byte)
}

__global__ void __launch_bounds__(kScoreTreeThreads) score_docs_tree_kernel(const __grid_constant__ ScoreDocsTreeLaunch L) {
  __shared__ ScoreTreeSmem sm;
  const int q = blockIdx.x / L.n_chunks, chunk = blockIdx.x % L.n_chunks;
  const int tid = threadIdx.x;
  if (tid == 0) { sm.q = L.queries[q]; sm.n_nodes = L.node_begin[q + 1] - L.node_begin[q]; }
  __syncthreads();
  const int ncl = sm.q.n_clauses;
  const int n_phrases = L.phrase_begin[q + 1] - L.phrase_begin[q];
  if (tid < ncl) sm.cl[tid] = L.clauses[sm.q.clause_begin + tid];
  if (tid < sm.n_nodes) sm.nodes[tid] = L.nodes[L.node_begin[q] + tid];
  if (tid < n_phrases) sm.phrases[tid] = L.phrases[L.phrase_begin[q] + tid];
  __syncthreads();
  for (int i = tid; i < ncl * 256; i += kScoreTreeThreads) {
    const int c = i >> 8;
    if (sm.cl[c].kind == NRTGPU_TERM) sm.cache[sm.cl[c].slot][i & 255] = L.ix.caches[sm.cl[c].field * 256 + (i & 255)];
  }
  __syncthreads();
  const int r = chunk * kScoreTreeThreads + tid;
  if (r >= L.n_hits) return;
  const size_t i = (size_t)q * L.n_hits + r;
  uint8_t m = 0; float s = 0.0f;
  if (!sm.q.empty && r < (L.counts ? L.counts[q] : L.n_hits)) {
    const int64_t local = (int64_t)L.docs[i] - L.ix.doc_base;
    if (local >= 0 && local < L.ix.n_docs) {
      const int32_t doc = (int32_t)local;
      uint64_t word = 0;   // the doc's tf byte of every term slot, as the window engine's pass 1 leaves it
      for (int c = 0; c < ncl; ++c) {
        const DevClause& cl = sm.cl[c];
        if (cl.kind != NRTGPU_TERM) continue;
        word |= (uint64_t)slot_lookup(L.ix, cl, doc, &sm.post[cl.slot][tid]) << (8 * cl.slot);
      }
      float sc;
      if (eval_tree(L.ix, sm, doc, word, &sc)) { m = 1; s = sc; }
    }
  }
  L.out_matches[i] = m; L.out_scores[i] = s;
}

// fetch phase: doc values of n_cols columns for n docs
struct FetchLaunch {
  DevIndexView ix;
  const int32_t* col_ids; int32_t n_cols;
  const int32_t* docs; int32_t n;   // global doc ids
  int64_t* out_values;              // [n_cols][n]
  uint8_t* out_has;                 // [n_cols][n]
};
__global__ void fetch_columns_kernel(FetchLaunch F) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)F.n_cols * F.n) return;
  const int c = F.col_ids[i / F.n];
  const int64_t local = (int64_t)F.docs[i % F.n] - F.ix.doc_base;
  int64_t v = 0; uint8_t h = 0;
  if (local >= 0 && local < F.ix.n_docs) {
    const uint8_t* has = F.ix.col_has[c];
    h = (!has || has[local]) ? 1 : 0;
    if (h) v = F.ix.col32[c] ? (int64_t)F.ix.col32[c][local] : F.ix.col64[c][local];
  }
  F.out_values[i] = v; F.out_has[i] = h;
}

// ---- aggregations over ALL matching docs of every query (ScoreMode.COMPLETE, as RelevanceCollector.java:55-62 forces)
// value types of a column (how the sortable long maps to the double the Min/Max/Sum collectors see)
enum { kAggInt = 0, kAggFloat = 1, kAggDouble = 2 };
__device__ __forceinline__ double agg_value(int64_t v, int value_type) {
  if (value_type == kAggFloat) { int32_t b = (int32_t)v; b ^= (b >> 31) & 0x7fffffff; return (double)__int_as_float(b); }   // NumericUtils.sortableIntToFloat
  if (value_type == kAggDouble) { long long b = v; b ^= (b >> 63) & 0x7fffffffffffffffll; return __longlong_as_double(b); }
  return (double)v;
}

struct AggSpecDev {
  int32_t kind;        // NRTGPU_AGG_*
  int32_t column, value_type;
  int32_t n_buckets;   // terms: distinct values of the column
  unsigned int* counts;        // terms: [nq][n_buckets]
  unsigned long long* dvals;   // min / max: ordered-double bits [nq]; sum: double bits [nq] (atomicAdd(double))
};
struct AggLaunch {
  AggSpecDev a[kMaxAggs];
  int32_t n_aggs;
  const uint32_t* codes[kMaxAggs];   // terms: sort codes of the column (bucket = code / 2 - 1)
};

__device__ __forceinline__ unsigned long long double_to_ordered(double d) {
  const unsigned long long b = (unsigned long long)__double_as_longlong(d);
  return (b & 0x8000000000000000ull) ? ~b : (b | 0x8000000000000000ull);
}
__host__ __device__ __forceinline__ double ordered_to_double(unsigned long long u) {
  const unsigned long long b = (u & 0x8000000000000000ull) ? (u & 0x7fffffffffffffffull) : ~u;
  double d;
#ifdef __CUDA_ARCH__
  d = __longlong_as_double((long long)b);
#else
  memcpy(&d, &b, sizeof(d));
#endif
  return d;
}

// called by the posting kernels for every matching doc of query q
__device__ __forceinline__ void agg_collect(const AggLaunch& A, const DevIndexView& ix, int q, int32_t doc) {
  for (int i = 0; i < A.n_aggs; ++i) {
    const AggSpecDev& s = A.a[i];
    const uint8_t* has = ix.col_has[s.column];
    if (has && !has[doc]) continue;   // LoadedDocValues.size() == 0: nothing to collect for this doc
    if (s.kind == NRTGPU_AGG_TERMS) {
      const uint32_t code = A.codes[i][doc];
      if (code) atomicAdd(&s.counts[(size_t)q * s.n_buckets + (code >> 1) - 1], 1u);
    } else {
      const int64_t raw = ix.col32[s.column] ? (int64_t)ix.col32[s.column][doc] : ix.col64[s.column][doc];
      const double v = agg_value(raw, s.value_type);
      // Max/MinCollectorManager keep `value > maxValue` (`value < minValue`) started from -/+Double.MAX_VALUE: NaN and the
      // infinity on the unset side never win
      if (s.kind == NRTGPU_AGG_MAX) { if (v > -DBL_MAX) atomicMax(&s.dvals[q], double_to_ordered(v)); }
      else if (s.kind == NRTGPU_AGG_MIN) { if (v < DBL_MAX) atomicMin(&s.dvals[q], double_to_ordered(v)); }
      else atomicAdd(reinterpret_cast<double*>(&s.dvals[q]), v);
    }
  }
}

// terms aggregation result of one query: the `size` buckets with the largest (or smallest) counts
// (TermsCollectorManager.fillBucketResultByCount :430-480), bucket keys as column values
struct AggTermsLaunch {
  const unsigned int* counts; int32_t n_buckets, nq, size, order_desc;
  const uint64_t* distinct;   // sorted distinct values (sortable u64) of the column
  int64_t* out_keys; int32_t* out_counts;   // [nq][size]
  int32_t* out_n;             // [nq] buckets returned
  int32_t* out_total_buckets; // [nq] non-empty buckets
  long long* out_other;       // [nq] docs counted in buckets not returned
};
__global__ void __launch_bounds__(256) agg_terms_topk_kernel(AggTermsLaunch T) {
  __shared__ uint64_t keys[2 * kAggChunk];
  __shared__ unsigned long long sh_sum;
  __shared__ int sh_nonzero;
  const int q = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) { sh_sum = 0ull; sh_nonzero = 0; }
  __syncthreads();
  const unsigned int* row = T.counts + (size_t)q * T.n_buckets;
  int have = 0;
  unsigned long long my_sum = 0; int my_nz = 0;
  for (int base = 0; base < T.n_buckets; base += kAggChunk) {
    for (int i = tid; i < kAggChunk; i += 256) {
      const int bkt = base + i;
      uint64_t k = 0ull;
      if (bkt < T.n_buckets) {
        const unsigned int c = row[bkt];
        if (c) {
          ++my_nz; my_sum += c;
          const uint32_t hi = T.order_desc ? c : ~c;                  // larger key = earlier bucket
          k = ((uint64_t)hi << 32) | (uint32_t)(~(uint32_t)bkt);        // ties: smaller value first (the reference leaves ties unordered)
        }
      }
      keys[have + i] = k;
    }
    const int n = have + kAggChunk;
    const int m = next_pow2(n);
    for (int i = n + tid; i < m; i += 256) keys[i] = 0ull;
    __syncthreads();
    block_bitonic_sort_desc(keys, m);
    have = min(T.size, kAggChunk);
    __syncthreads();
  }
  atomicAdd(&sh_sum, my_sum); atomicAdd(&sh_nonzero, my_nz);
  __syncthreads();
  int n_out = 0;
  unsigned long long shown = 0;
  for (int i = 0; i < have; ++i) if (keys[i]) ++n_out; else break;   // (uniform: every thread scans the same smem)
  for (int i = tid; i < T.size; i += 256) {
    int64_t key = 0; int32_t cnt = 0;
    if (i < n_out) {
      const uint32_t hi = (uint32_t)(keys[i] >> 32), bkt = ~(uint32_t)keys[i];
      cnt = (int32_t)(T.order_desc ? hi : ~hi);
      key = (int64_t)(T.distinct[bkt] ^ 0x8000000000000000ull);
    }
    T.out_keys[(size_t)q * T.size + i] = key; T.out_counts[(size_t)q * T.size + i] = cnt;
  }
  if (tid == 0) {
    for (int i = 0; i < n_out; ++i) { const uint32_t hi = (uint32_t)(keys[i] >> 32); shown += T.order_desc ? hi : ~hi; }
    T.out_n[q] = n_out; T.out_total_buckets[q] = sh_nonzero; T.out_other[q] = (long long)(sh_sum - shown);
  }
}

}  // namespace nrtgpu
