// Per-query filter queries of the kNN path (KnnQuery.filter, reference src/main/java/com/yelp/nrtsearch/server/search/
// KnnUtils.java:135-155), evaluated on the device into one bitmap row per distinct filter of a call:
// uint32[n_rows][ceil(n_docs / 32)], bit d set iff live doc d matches the filter. Rows are built word-parallel:
//   * a term clause reads the bitmap of its term, built once per call by scattering the term's postings (cost ~ df);
//   * a range clause runs range_matches (a keyword range keyword_matches) with one lane per doc, a warp ballot forms the word;
//   * match-all is ~0;
//   * the words combine as eval_clauses (query_eval.cuh) matches: AND of MUST / FILTER, minus the OR of MUST_NOT, and at least
//     need_should SHOULD clauses per bit (a bit-sliced counter); an empty query gives 0.
// The kNN stages then AND bit d of the query's row into their filter test (knn_gemm_tc.cuh, knn_kernel.cuh), and the
// queries whose row is small are scored exactly over the row's ordinals only (knn_filter_ords_kernel + the gather mode of
// knn_exact_chunk_kernel).
#pragma once
#include "query_eval.cuh"

namespace nrtgpu {

// A query whose filter matches c <= n_vec / kKnnGatherRatio docs is scored exactly over those docs' vectors (c gathered
// vectors, fp64) instead of going through the candidate GEMM over all n_vec (DESIGN.md §4.3 gives the H100 measurements).
constexpr int64_t kKnnGatherRatio = 320;
// Fixed scratch budget of the filter evaluation: the rows of one call are capped at kKnnFilterRowBytes (a call with more
// distinct filters runs in groups of queries whose rows fit), and the term bitmaps built at once at kKnnFilterTermBytes
// (the filters of a group are evaluated in subgroups whose terms fit). A group holds at least one row and a subgroup one
// filter's terms, which exceed the budget on their own only past 2^30 docs (a row) or 2^27 docs (8 term bitmaps).
constexpr size_t kKnnFilterRowBytes = (size_t)128 << 20;
constexpr size_t kKnnFilterTermBytes = (size_t)128 << 20;

struct KnnTermScatterLaunch {
  const int32_t* post_docs;
  const int64_t* term_base;   // [n_terms] offset of each distinct term's postings in post_docs
  const int64_t* term_pre;    // [n_terms + 1] running sum of the terms' posting counts
  int n_terms, words;
  uint32_t* tbits;            // [n_terms][words], zeroed
};

// one thread per posting of the group's distinct terms: sets the doc's bit in its term's bitmap
__global__ void __launch_bounds__(256) knn_term_scatter_kernel(KnnTermScatterLaunch L) {
  const int64_t p0 = L.term_pre[0], p1 = L.term_pre[L.n_terms];
  for (int64_t i = p0 + blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < p1; i += (int64_t)gridDim.x * blockDim.x) {
    int lo = 0, hi = L.n_terms;   // the term of posting i: the last t with term_pre[t] <= i
    while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (L.term_pre[m] <= i) lo = m; else hi = m; }
    const int32_t doc = __ldg(L.post_docs + L.term_base[lo] + (i - L.term_pre[lo]));
    atomicOr(L.tbits + (size_t)lo * L.words + (doc >> 5), 1u << (doc & 31));
  }
}

struct KnnFilterRowsLaunch {
  DevIndexView ix;
  const DevClause* clauses; const DevQuery* filters;   // the compiled filters (batch_build)
  const int32_t* row_filter;    // [n_rows] filter of each row
  const int32_t* clause_term;   // [n_clauses] term clause: its term's bitmap in tbits (-1: the term has no postings)
  const uint32_t* tbits;        // [group terms][words]
  int row0, words;              // rows row0 + blockIdx.y
  uint32_t* rows;               // [n_rows][words]
  int32_t* row_cnt;             // [n_rows] matching docs, zeroed
};

// word w0 + lane of a keyword range clause's row, as the range branch of knn_filter_rows_kernel forms it: for word w0 + j
// lane l tests doc 32 (w0 + j) + l, a warp ballot forms the word (out of line: inlined, it makes the kernel spill)
__device__ __noinline__ uint32_t keyword_row_word(const uint32_t* codes, const int64_t* off, int32_t n_docs, int64_t lo, int64_t hi,
                                                  int w0, int lane) {
  uint32_t x = 0u;
  for (int j = 0; j < 32; ++j) {
    const int64_t doc = 32ll * (w0 + j) + lane;
    const bool m = doc < n_docs && keyword_codes_match(codes, off, (int32_t)doc, lo, hi);
    const uint32_t b = __ballot_sync(0xffffffffu, m);
    if (lane == j) x = b;
  }
  return x;
}

// one thread per (row, word); a warp covers 32 consecutive words of one row
__global__ void __launch_bounds__(256) knn_filter_rows_kernel(KnnFilterRowsLaunch L) {
  const int row = L.row0 + blockIdx.y, lane = threadIdx.x & 31;
  const int w = blockIdx.x * blockDim.x + threadIdx.x, w0 = w - lane;
  const DevQuery& q = L.filters[L.row_filter[row]];
  uint32_t req = ~0u, excl = 0u, cnt[5] = {0u, 0u, 0u, 0u, 0u};
  for (int i = 0; i < q.n_clauses; ++i) {
    const DevClause& c = L.clauses[q.clause_begin + i];
    uint32_t x = 0u;
    if (c.kind == NRTGPU_TERM) {
      const int t = L.clause_term[q.clause_begin + i];
      if (t >= 0 && w < L.words) x = L.tbits[(size_t)t * L.words + w];
    } else if (c.kind == NRTGPU_RANGE_I64) {
      for (int j = 0; j < 32; ++j) {   // word w0 + j: lane l tests doc 32 (w0 + j) + l
        const int64_t doc = 32ll * (w0 + j) + lane;
        const bool m = doc < L.ix.n_docs && range_matches(L.ix, c.col, (int32_t)doc, c.lo, c.hi);
        const uint32_t b = __ballot_sync(0xffffffffu, m);
        if (lane == j) x = b;
      }
    } else if (c.kind == NRTGPU_KEYWORD_RANGE) {
      x = keyword_row_word(L.ix.kw_codes[c.col], L.ix.kw_off[c.col], L.ix.n_docs, c.lo, c.hi, w0, lane);
    } else {
      x = ~0u;
    }
    if (c.occur == NRTGPU_MUST || c.occur == NRTGPU_FILTER) req &= x;
    else if (c.occur == NRTGPU_MUST_NOT) excl |= x;
    else {   // SHOULD: add x to the 5-bit counter (at most 16 clauses)
      uint32_t carry = x;
#pragma unroll
      for (int b = 0; b < 5; ++b) { const uint32_t t = cnt[b] & carry; cnt[b] ^= carry; carry = t; }
    }
  }
  // count >= need_should, compared bit-sliced from the most significant bit down
  uint32_t gt = 0u, eq = ~0u;
#pragma unroll
  for (int b = 4; b >= 0; --b) {
    if ((q.need_should >> b) & 1) eq &= cnt[b];
    else { gt |= eq & cnt[b]; eq &= ~cnt[b]; }
  }
  uint32_t word = 0u;
  if (w < L.words && !q.empty) {
    word = req & ~excl & (gt | eq);
    if (L.ix.live_bits) word &= L.ix.live_bits[w];
    const int tail = L.ix.n_docs - 32 * w;
    if (tail < 32) word &= (1u << tail) - 1u;
  }
  if (w < L.words) L.rows[(size_t)row * L.words + w] = word;
  int n = __popc(word);
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
  if (lane == 0 && n) atomicAdd(L.row_cnt + row, n);
}

// The row of a filter collector's value set (FilterCollectorManager.SetQueryFilter over a TermInSetQuery): bit d is set iff
// live doc d has a value of `column` in set[0 .. n_set), sorted and distinct in the column's sortable-long domain, so a
// match is bit equality (-0.0 != 0.0, NaN == NaN, as Java's boxed equals). One lane per doc and a warp ballot per word, as
// the range branch above; a multi-valued doc passes when any of its values is in the set. A keyword set
// (NRTGPU_AGG_FILTER_KEYWORD_SET) holds codes of keyword column `column`: a doc passes when one of its terms' codes is in
// it (a set holds no code 0, so a doc without a value never passes).
struct AggValueSetLaunch {
  DevIndexView ix;
  int32_t column, n_set, words, keyword;
  const int64_t* set;
  uint32_t* row;   // [words]
};

__device__ __forceinline__ bool in_sorted_set(const int64_t* __restrict__ set, int n, int64_t v) {
  int lo = 0, hi = n;
  while (lo < hi) { const int m = (lo + hi) >> 1; if (__ldg(set + m) < v) lo = m + 1; else hi = m; }
  return lo < n && __ldg(set + lo) == v;
}

__global__ void __launch_bounds__(256) agg_value_set_kernel(AggValueSetLaunch L) {
  const int64_t doc = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool m = false;
  if (doc < L.ix.n_docs && L.n_set > 0) {
    const int32_t d = (int32_t)doc;
    const int64_t* off = L.keyword ? L.ix.kw_off[L.column] : L.ix.colmv_off ? L.ix.colmv_off[L.column] : nullptr;
    if (L.keyword) {
      const uint32_t* v = L.ix.kw_codes[L.column];
      if (off) for (int64_t j = off[d]; j < off[d + 1] && !m; ++j) m = in_sorted_set(L.set, L.n_set, (int64_t)__ldg(v + j));
      else m = in_sorted_set(L.set, L.n_set, (int64_t)__ldg(v + d));
    } else if (off) {
      const int64_t* v = L.ix.colmv_val[L.column];
      for (int64_t j = off[d]; j < off[d + 1] && !m; ++j) m = in_sorted_set(L.set, L.n_set, v[j]);
    } else {
      const uint8_t* has = L.ix.col_has[L.column];
      if (!has || has[d])
        m = in_sorted_set(L.set, L.n_set, L.ix.col32[L.column] ? (int64_t)__ldg(L.ix.col32[L.column] + d) : __ldg(L.ix.col64[L.column] + d));
    }
  }
  uint32_t word = __ballot_sync(0xffffffffu, m);
  const int64_t w = doc >> 5;
  if ((threadIdx.x & 31) == 0 && w < L.words) {
    if (L.ix.live_bits) word &= L.ix.live_bits[w];
    L.row[w] = word;
  }
}

// a filter nested under a filter: its row ANDs its parent's
__global__ void row_and_kernel(uint32_t* __restrict__ dst, const uint32_t* __restrict__ src, int words) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < words) dst[i] &= src[i];
}

// The codes a filter collector's aggregation counts through in agg_collect, which sees it as a terms aggregation: a filter
// is one bucket (code 2) where its row passes, and a terms aggregation under a filter keeps its column's codes (src) there;
// 0 (no bucket) elsewhere
__global__ void agg_row_codes_kernel(const uint32_t* __restrict__ row, const uint32_t* __restrict__ src, int32_t n_docs,
                                     uint32_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_docs) return;
  out[i] = ((row[i >> 5] >> (i & 31)) & 1u) ? (src ? src[i] : 2u) : 0u;
}

// agg_row_codes_kernel for a terms aggregation over a SORTED_SET keyword column: each value of a doc keeps its code (src,
// value-indexed through the doc offsets off) where the doc's row passes, 0 elsewhere
__global__ void agg_row_value_codes_kernel(const uint32_t* __restrict__ row, const uint32_t* __restrict__ src,
                                           const int64_t* __restrict__ off, int32_t n_docs, uint32_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_docs) return;
  const bool pass = (row[i >> 5] >> (i & 31)) & 1u;
  for (int64_t v = off[i]; v < off[i + 1]; ++v) out[v] = pass ? src[v] : 0u;
}

struct KnnFilterOrdsLaunch {
  const uint32_t* rows; int words;
  const int32_t* grows;         // rows to compact: grows[blockIdx.y]
  const int64_t* ord_begin;     // [n_rows] start of each row's list in ords (row_cnt[r] entries reserved)
  const int32_t* vec_docs;      // ordinal -> doc or NULL (identity)
  int n_vec;
  int32_t* ords; int32_t* ord_cnt;   // [n_rows] ordinals listed, zeroed
};

// The ordinals whose doc is set in the row, in no particular order (the exact scorer's top-k sort is total). Without
// vec_docs the ordinals are the set bits below n_vec: one thread per word; with it every ordinal is tested.
__global__ void __launch_bounds__(256) knn_filter_ords_kernel(KnnFilterOrdsLaunch L) {
  const int row = L.grows[blockIdx.y], lane = threadIdx.x & 31;
  const uint32_t* r = L.rows + (size_t)row * L.words;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t bits = 0u;   // ordinals this thread lists: bit b = ordinal base + b
  int base = 0;
  if (!L.vec_docs) {
    base = 32 * i;
    if (base < L.n_vec) {
      bits = r[i];
      if (L.n_vec - base < 32) bits &= (1u << (L.n_vec - base)) - 1u;
    }
  } else if (i < L.n_vec) {
    const int doc = L.vec_docs[i];
    base = i;
    bits = (r[doc >> 5] >> (doc & 31)) & 1u;
  }
  const int n = __popc(bits);
  int incl = n;   // warp-inclusive prefix of the counts: one atomic per warp
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  int pos = 0;
  if (lane == 31 && incl) pos = atomicAdd(L.ord_cnt + row, incl);
  pos = __shfl_sync(0xffffffffu, pos, 31) + incl - n;
  int32_t* out = L.ords + L.ord_begin[row] + pos;
  while (bits) { const int b = __ffs(bits) - 1; bits &= bits - 1; *out++ = base + b; }
}

}  // namespace nrtgpu
