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
// a nested collector of a terms aggregation, at the parent's (query, bucket) cell
struct AggNestedDev {
  int32_t kind;                 // NRTGPU_AGG_MIN / _MAX / _SUM (pass 1) or NRTGPU_AGG_TOP_HITS (pass 2)
  int32_t column, value_type;   // MIN / MAX / SUM
  int32_t size;                 // TOP_HITS: the parent's size (slots per query)
  int32_t q_lo, q_hi;           // TOP_HITS: the queries of this pass-2 group
  int32_t doc_base;             // TOP_HITS: the image's first global doc (keys of several leaves share the segments)
  unsigned long long* dvals;    // MIN / MAX / SUM: [nq][n_buckets] words as AggSpecDev::dvals
  const int32_t* slot_of;       // TOP_HITS: [nq][n_buckets] returned slot of the bucket, -1: not returned
  const long long* hit_off;     // TOP_HITS: [q_hi - q_lo][size] first key of the (query, slot)
  unsigned int* hit_fill;       // TOP_HITS: [q_hi - q_lo][size] keys written
  uint64_t* hit_keys;           // TOP_HITS: make_key(score, global doc) of the collected docs, or their Sort keys (rank)
  const uint32_t* rank;         // TOP_HITS by a Sort: the order's rank of each doc of the image (NULL: by score)
  int32_t score_key;            // TOP_HITS: the key's high word is the ordered score (by score, or a Sort led by SCORE) ...
  int32_t score_reverse;        // ... negated (a reversed leading SCORE: lower scores first)
};
struct AggLaunch {
  AggSpecDev a[kMaxAggs];
  int32_t n_aggs;
  const uint32_t* codes[kMaxAggs];   // terms: sort codes of the column (bucket = code / 2 - 1)
  int32_t nested_begin[kMaxAggs + 1];   // terms: nested[nested_begin[i], nested_begin[i + 1]) are aggregation i's
  AggNestedDev nested[kMaxAggs * kMaxNested];
  // terms over a SORTED_SET keyword column (read by the kMulti instantiations only; last, so that the other members keep
  // their offsets): doc d's value codes are codes[i][offsets[i][d], offsets[i][d + 1]); NULL: one code per doc
  const int64_t* offsets[kMaxAggs];
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

// a min / max / sum collector's word takes the doc's value in `column`, if it has one
__device__ __forceinline__ void agg_metric_collect(int kind, int column, int value_type, unsigned long long* w,
                                                   const DevIndexView& ix, int32_t doc) {
  const uint8_t* has = ix.col_has[column];
  if (has && !has[doc]) return;   // LoadedDocValues.size() == 0: nothing to collect for this doc
  const int64_t raw = ix.col32[column] ? (int64_t)ix.col32[column][doc] : ix.col64[column][doc];
  const double v = agg_value(raw, value_type);
  // Max/MinCollectorManager keep `value > maxValue` (`value < minValue`) started from -/+Double.MAX_VALUE: NaN and the
  // infinity on the unset side never win
  if (kind == NRTGPU_AGG_MAX) { if (v > -DBL_MAX) atomicMax(w, double_to_ordered(v)); }
  else if (kind == NRTGPU_AGG_MIN) { if (v < DBL_MAX) atomicMin(w, double_to_ordered(v)); }
  else atomicAdd(reinterpret_cast<double*>(w), v);
}

// the nested collectors of a terms aggregation for a doc counted in bucket cell (q * n_buckets + bucket)
__device__ __noinline__ void agg_nested_collect(const AggLaunch& A, int i, const DevIndexView& ix, int q, size_t cell,
                                                int32_t doc, float score) {
  for (int j = A.nested_begin[i]; j < A.nested_begin[i + 1]; ++j) {
    const AggNestedDev& n = A.nested[j];
    if (n.kind != NRTGPU_AGG_TOP_HITS) { agg_metric_collect(n.kind, n.column, n.value_type, n.dvals + cell, ix, doc); continue; }
    if (q < n.q_lo || q >= n.q_hi) continue;
    const int slot = n.slot_of[cell];
    if (slot < 0) continue;
    const size_t s = (size_t)(q - n.q_lo) * n.size + slot;
    // by score make_key(score, global doc); by a Sort a key whose descending order is the Sort's: ~rank (unique, 1-based, it
    // holds the doc tie-break), under a leading SCORE the ordered score above it, flipped for reverse (kSortScoreRank's key)
    const uint32_t lo = n.rank ? n.rank[doc] : (uint32_t)(doc + n.doc_base);
    const uint32_t hi = n.score_key ? float_to_ordered(n.score_reverse ? -score : score) : 0u;
    n.hit_keys[n.hit_off[s] + atomicAdd(&n.hit_fill[s], 1u)] = ((uint64_t)hi << 32) | (uint32_t)~lo;   // sized by the bucket's count
  }
}

// terms aggregation i over a SORTED_SET keyword column for a matching doc: the doc counts once in the bucket of each of its
// terms and is handed to the nested collectors once per term (OrdinalTermsCollectorManager: nestedLeafCollectors.collect(
// globalOrd, doc) per ord). A doc's terms are distinct, so no bucket sees a doc twice.
__device__ __forceinline__ void agg_collect_values(const AggLaunch& A, int i, const DevIndexView& ix, int q, int32_t doc, float score) {
  const AggSpecDev& s = A.a[i];
  const bool nested = A.nested_begin[i + 1] > A.nested_begin[i];
  const uint32_t* codes = A.codes[i];
  for (int64_t v = A.offsets[i][doc], e = A.offsets[i][doc + 1]; v < e; ++v) {
    const uint32_t code = codes[v];
    if (!code) continue;   // (a value whose doc a filter's row gates out)
    const size_t cell = (size_t)q * s.n_buckets + (code >> 1) - 1;
    if (s.counts) atomicAdd(&s.counts[cell], 1u);   // (NULL in the top-hits run)
    if (nested) agg_nested_collect(A, i, ix, q, cell, doc, score);
  }
}

// called by the posting kernels for every matching doc of query q (score: its score under a relevance sort). kMulti: the
// launch carries a SORTED_SET keyword terms aggregation (A.offsets); only the kMulti kernel instantiations read A.offsets,
// so the others run the code they ran before keyword columns.
template <bool kMulti = false>
__device__ __forceinline__ void agg_collect(const AggLaunch& A, const DevIndexView& ix, int q, int32_t doc, float score) {
  for (int i = 0; i < A.n_aggs; ++i) {
    const AggSpecDev& s = A.a[i];
    if (s.kind == NRTGPU_AGG_TERMS) {
      const uint8_t* has = ix.col_has[s.column];
      if (has && !has[doc]) continue;
      if constexpr (kMulti) {
        if (A.offsets[i]) { agg_collect_values(A, i, ix, q, doc, score); continue; }
      }
      const uint32_t code = A.codes[i][doc];
      if (!code) continue;
      const size_t cell = (size_t)q * s.n_buckets + (code >> 1) - 1;
      if (s.counts) atomicAdd(&s.counts[cell], 1u);   // (NULL in the top-hits run)
      if (A.nested_begin[i + 1] > A.nested_begin[i]) agg_nested_collect(A, i, ix, q, cell, doc, score);
    } else {
      agg_metric_collect(s.kind, s.column, s.value_type, &s.dvals[q], ix, doc);
    }
  }
}

// ---- reader-wide value dictionary of a searcher over several leaves: every leaf numbers a column's values in its own
// dictionary (col_distinct, col_code), so a leaf's codes are renumbered to the sorted union of the leaves' dictionaries,
// whose bucket g is code 2g + 2 in every leaf. Union order is value order, so the selection's tie rules hold unchanged.
// the reader-wide bucket of each bucket of a leaf: the position of its value in the union (where it is present)
__global__ void dict_map_kernel(const uint64_t* __restrict__ leaf, int32_t n_leaf, const uint64_t* __restrict__ uni, int32_t n_uni,
                                uint32_t* __restrict__ map) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_leaf) return;
  const uint64_t v = leaf[i];
  int lo = 0, hi = n_uni;
  while (lo < hi) { const int m = (lo + hi) >> 1; if (uni[m] < v) lo = m + 1; else hi = m; }
  map[i] = (uint32_t)lo;
}
// a leaf's codes through that map: 2b + 2 -> 2 map[b] + 2; 0 (no value) stays 0
__global__ void dict_remap_kernel(const uint32_t* __restrict__ codes, int64_t n, const uint32_t* __restrict__ map, uint32_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t c = codes[i];
  out[i] = c ? 2u * map[(c >> 1) - 1] + 2u : 0u;
}

// the double a min / max / sum word stands for, the collectors' unset value where no doc had a value
__host__ __device__ __forceinline__ double agg_word_value(int kind, unsigned long long w) {
  if (kind == NRTGPU_AGG_SUM) {
    double v;
#ifdef __CUDA_ARCH__
    v = __longlong_as_double((long long)w);
#else
    memcpy(&v, &w, sizeof(v));
#endif
    return v;
  }
  if (kind == NRTGPU_AGG_MAX) return w == 0ull ? -DBL_MAX : ordered_to_double(w);   // MaxCollectorManager.UNSET_VALUE
  return w == ~0ull ? DBL_MAX : ordered_to_double(w);                                // MinCollectorManager.UNSET_VALUE
}

// terms aggregation result of one query: the `size` buckets with the largest (or smallest) counts
// (TermsCollectorManager.fillBucketResultByCount :430-480), bucket keys as column values
struct AggTermsLaunch {
  const unsigned int* counts; int32_t n_buckets, nq, size, order_desc;
  const uint64_t* distinct;   // sorted distinct values (sortable u64) of the column; NULL: keys are the buckets (keyword ordinals)
  int64_t* out_keys; int32_t* out_counts;   // [nq][size]
  int32_t* out_n;             // [nq] buckets returned
  int32_t* out_total_buckets; // [nq] non-empty buckets
  long long* out_other;       // [nq] docs counted in buckets not returned
  int32_t* out_bucket;        // optional [nq][size] bucket of each returned slot, -1 past out_n (nested collectors)
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
      key = T.distinct ? (int64_t)(T.distinct[bkt] ^ 0x8000000000000000ull) : (int64_t)bkt;
    }
    T.out_keys[(size_t)q * T.size + i] = key; T.out_counts[(size_t)q * T.size + i] = cnt;
    if (T.out_bucket) T.out_bucket[(size_t)q * T.size + i] = i < n_out ? (int32_t)~(uint32_t)keys[i] : -1;
  }
  if (tid == 0) {
    for (int i = 0; i < n_out; ++i) { const uint32_t hi = (uint32_t)(keys[i] >> 32); shown += T.order_desc ? hi : ~hi; }
    T.out_n[q] = n_out; T.out_total_buckets[q] = sh_nonzero; T.out_other[q] = (long long)(sh_sum - shown);
  }
}

// In-place bitonic sort of n (power of two) (key, tag) pairs in shared memory by the whole CTA, descending by key, then tag.
__device__ __forceinline__ void block_bitonic_sort_pairs_desc(uint64_t* a, uint32_t* t, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
        const int lo = ((i & ~(j - 1)) << 1) | (i & (j - 1)), hi = lo | j;
        const bool desc = (lo & k) == 0;
        const uint64_t x = a[lo], y = a[hi];
        const uint32_t tx = t[lo], ty = t[hi];
        if ((x < y || (x == y && tx < ty)) == desc) { a[lo] = y; a[hi] = x; t[lo] = ty; t[hi] = tx; }
      }
      __syncthreads();
    }
  }
}

// terms aggregation ordered by a nested min / max / sum (TermsCollectorManager.fillBucketResultByNestedOrder :930-994): the
// `size` non-empty buckets whose value is largest (order_desc) or smallest by Double.compare, ties to the smaller bucket
// value. Outputs as agg_terms_topk_kernel. Dynamic shared memory: kAggByValueSmem.
constexpr int kAggByValueSmem = 2 * kAggChunk * (int)(sizeof(uint64_t) + sizeof(uint32_t));
__global__ void __launch_bounds__(256) agg_terms_by_value_kernel(AggTermsLaunch T, const unsigned long long* words, int kind) {
  extern __shared__ uint64_t dyn_keys[];
  uint64_t* keys = dyn_keys;                                    // the value's Double.compare order (flipped for ASC)
  uint32_t* tags = reinterpret_cast<uint32_t*>(dyn_keys + 2 * kAggChunk);   // ~bucket; 0: no bucket
  __shared__ unsigned long long sh_sum;
  __shared__ int sh_nonzero;
  const int q = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) { sh_sum = 0ull; sh_nonzero = 0; }
  __syncthreads();
  const unsigned int* row = T.counts + (size_t)q * T.n_buckets;
  const unsigned long long* wrow = words + (size_t)q * T.n_buckets;
  int have = 0;
  unsigned long long my_sum = 0; int my_nz = 0;
  for (int base = 0; base < T.n_buckets; base += kAggChunk) {
    for (int i = tid; i < kAggChunk; i += 256) {
      const int bkt = base + i;
      uint64_t k = 0ull; uint32_t g = 0u;
      if (bkt < T.n_buckets) {
        const unsigned int c = row[bkt];
        if (c) {   // the reference's counts map holds the buckets with a doc
          ++my_nz; my_sum += c;
          double v = agg_word_value(kind, wrow[bkt]);
          if (v != v) v = __longlong_as_double(0x7ff8000000000000ll);   // Double.compare: every NaN above +inf
          const uint64_t o = double_to_ordered(v);
          k = T.order_desc ? o : ~o;
          g = ~(uint32_t)bkt;
        }
      }
      keys[have + i] = k; tags[have + i] = g;
    }
    const int n = have + kAggChunk;
    const int m = next_pow2(n);
    for (int i = n + tid; i < m; i += 256) { keys[i] = 0ull; tags[i] = 0u; }
    __syncthreads();
    block_bitonic_sort_pairs_desc(keys, tags, m);
    have = min(T.size, kAggChunk);
    __syncthreads();
  }
  atomicAdd(&sh_sum, my_sum); atomicAdd(&sh_nonzero, my_nz);
  __syncthreads();
  int n_out = 0;
  for (int i = 0; i < have; ++i) if (tags[i]) ++n_out; else break;
  for (int i = tid; i < T.size; i += 256) {
    int64_t key = 0; int32_t cnt = 0, bkt = -1;
    if (i < n_out) {
      bkt = (int32_t)~tags[i];
      cnt = (int32_t)row[bkt];
      key = T.distinct ? (int64_t)(T.distinct[bkt] ^ 0x8000000000000000ull) : (int64_t)bkt;
    }
    T.out_keys[(size_t)q * T.size + i] = key; T.out_counts[(size_t)q * T.size + i] = cnt;
    if (T.out_bucket) T.out_bucket[(size_t)q * T.size + i] = bkt;
  }
  if (tid == 0) {
    unsigned long long shown = 0;
    for (int i = 0; i < n_out; ++i) shown += row[~tags[i]];
    T.out_n[q] = n_out; T.out_total_buckets[q] = sh_nonzero; T.out_other[q] = (long long)(sh_sum - shown);
  }
}

// per returned slot of a terms aggregation: the slot map of its buckets (top hits) and its nested min / max / sum values
struct AggNestedOutLaunch {
  const int32_t* bucket;      // [nq][size] (out_bucket of the selection)
  int32_t nq, size, n_buckets;
  int32_t* slot_of;           // optional [nq][n_buckets], preset to -1
  int32_t n_vals;
  int32_t kind[kMaxNested];
  const unsigned long long* words[kMaxNested];   // [nq][n_buckets]
  double* values[kMaxNested];                    // [nq][size]; 0 past the returned buckets
};
__global__ void agg_nested_out_kernel(AggNestedOutLaunch O) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= O.nq * O.size) return;
  const int32_t b = O.bucket[i];
  const size_t cell = (size_t)(i / O.size) * O.n_buckets + b;
  if (O.slot_of && b >= 0) O.slot_of[cell] = i % O.size;
  for (int j = 0; j < O.n_vals; ++j) O.values[j][i] = b >= 0 ? agg_word_value(O.kind[j], O.words[j][cell]) : 0.0;
}

// nested top hits of the returned buckets of one pass-2 group: one CTA per (query, slot) keeps the best top_hits keys of
// its segment (a chunk is sorted only when one of its keys beats the current top_hits-th) and writes [start_hit, top_hits)
struct NestedHitsLaunch {
  const uint64_t* hit_keys;
  const long long* hit_off;     // [group * size + 1]
  const unsigned int* hit_fill; // [group * size]
  int32_t q_lo, size, top_hits, start_hit, doc_base;
  int32_t* out_docs; float* out_scores;   // [nq][size][top_hits - start_hit]
  int32_t* out_counts;                    // [nq][size]
};
__global__ void __launch_bounds__(256) nested_top_hits_kernel(NestedHitsLaunch H) {
  __shared__ uint64_t keys[2 * kAggChunk];   // the best (<= 1024) and a chunk's admitted keys
  __shared__ int sh_new;
  const int g = blockIdx.x, tid = threadIdx.x;
  const long long off = H.hit_off[g];
  const int n = (int)min((long long)H.hit_fill[g], H.hit_off[g + 1] - off);
  const uint64_t* src = H.hit_keys + off;
  int have = 0;
  uint64_t kth = 0ull;
  for (int base = 0; base < n; base += kAggChunk) {
    if (tid == 0) sh_new = 0;
    __syncthreads();
    for (int i = tid; i < kAggChunk; i += 256) {
      const int x = base + i;
      if (x < n) {
        const uint64_t k = src[x];
        if (have < H.top_hits || k > kth) keys[have + atomicAdd(&sh_new, 1)] = k;   // (keys are distinct: doc ids)
      }
    }
    __syncthreads();
    const int added = sh_new;
    __syncthreads();
    if (added == 0) continue;
    const int tot = have + added, m = next_pow2(tot < 2 ? 2 : tot);
    for (int i = tot + tid; i < m; i += 256) keys[i] = 0ull;
    __syncthreads();
    block_bitonic_sort_desc(keys, m);
    have = min(tot, H.top_hits);
    kth = keys[have - 1];
  }
  const int w = H.top_hits - H.start_hit;
  const size_t qs = (size_t)(H.q_lo + g / H.size) * H.size + g % H.size;
  for (int i = tid; i < w; i += 256) {
    const int p = H.start_hit + i;
    int32_t doc = 0; float score = 0.0f;
    if (p < have) { doc = key_doc(keys[p]) + H.doc_base; score = key_score(keys[p]); }
    H.out_docs[qs * w + i] = doc; H.out_scores[qs * w + i] = score;
  }
  if (tid == 0) H.out_counts[qs] = max(0, have - H.start_hit);
}

}  // namespace nrtgpu
