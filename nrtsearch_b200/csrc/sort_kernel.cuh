// Sort-by-field top-k (TopFieldCollector semantics; reference
// src/main/java/com/yelp/nrtsearch/server/search/collectors/SortFieldCollector.java:44-105, numeric sort fields
// .../field/NumberFieldDef.java:266-278, missing values IntFieldDef.java:103 / LongFieldDef.java:103 / ...).
//
// The top-k machinery of the posting kernels orders 64-bit keys (hi word desc, then ~doc desc = doc asc). A sorted
// search swaps the key function: hi = an ORDER-PRESERVING 32-bit code of the doc's sort value. The codes are index-time
// data, one uint32 per doc and column: the column's distinct values are sorted once on the device and value number i
// (0-based) gets code 2i + 2; code 2i + 1 stands for "between value i-1 and value i" (the code of a value the column
// does not hold: a missing_value such as Long.MIN_VALUE, or the searchAfter value of another shard). So any int64 can
// be compared with every doc exactly, ties included (a doc WITHOUT a value takes the code of missing_value at query
// time, and therefore ties with docs that really hold that value, as Lucene's comparator does).
#pragma once
#include <thrust/copy.h>
#include <thrust/execution_policy.h>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/scan.h>
#include <thrust/sequence.h>
#include <thrust/sort.h>
#include <thrust/system/cuda/execution_policy.h>
#include "common.cuh"

namespace nrtgpu {

__host__ __device__ __forceinline__ uint64_t sortable_u64(int64_t v) { return (uint64_t)v ^ 0x8000000000000000ull; }

struct SortNonZero { __host__ __device__ bool operator()(uint8_t x) const { return x != 0; } };

// keys[i] = sortable value of doc idx[i] (idx = the docs that have a value)
__global__ void sort_col_keys_kernel(const int64_t* __restrict__ c64, const int32_t* __restrict__ c32, const int32_t* __restrict__ idx,
                                     int32_t n, uint64_t* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t d = idx[i];
  keys[i] = sortable_u64(c32 ? (int64_t)c32[d] : c64[d]);
}
__global__ void sort_mark_kernel(const uint64_t* __restrict__ keys, int32_t n, int32_t* __restrict__ mark) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  mark[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}
// rank[i] = 1-based number of the distinct value of sorted position i
__global__ void sort_scatter_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ idx, const int32_t* __restrict__ rank,
                                    int32_t n, uint32_t* __restrict__ codes, uint64_t* __restrict__ distinct) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t r = rank[i] - 1;
  codes[idx[i]] = 2u * (uint32_t)r + 2u;
  if (i == 0 || keys[i] != keys[i - 1]) distinct[r] = keys[i];
}

// order-preserving code of an arbitrary value against a column's sorted distinct values
__device__ __forceinline__ uint32_t sort_code_of(const uint64_t* __restrict__ distinct, int32_t n_distinct, int64_t v) {
  const uint64_t k = sortable_u64(v);
  int lo = 0, hi = n_distinct;
  while (lo < hi) { const int m = (lo + hi) >> 1; if (distinct[m] < k) lo = m + 1; else hi = m; }
  return (lo < n_distinct && distinct[lo] == k) ? 2u * (uint32_t)lo + 2u : 2u * (uint32_t)lo + 1u;
}

struct SortAfterLaunch {
  DevQuery* queries; int32_t nq;
  const int32_t* after_docs;      // [nq] global doc ids (nrtgpu_query.after_doc)
  const int64_t* after_values;    // [nq]
  int32_t kind, reverse, doc_base, n_docs;
  const uint64_t* distinct; int32_t n_distinct;
  int64_t missing_value;
  uint32_t* missing_code;         // [1] out: code of missing_value
};

__device__ __forceinline__ uint32_t sort_hi(int kind, int reverse, uint32_t code, int32_t doc) {
  if (kind == NRTGPU_SORT_DOCID) return reverse ? (uint32_t)doc + 1u : 0x7fffffffu;
  return reverse ? code : ~code;
}

// patches DevQuery::after_key of every query with searchAfter: a hit qualifies iff key < after_key. An odd code is held by
// no doc, but the docs without a value carry the code of missing_value, which may be that same odd code: an after value
// equal to missing_value ties with them (the doc part decides, as for a held value); any other after value in the same
// gap between held values precedes all of them or follows all of them, by the order of the two values.
__global__ void sort_after_kernel(SortAfterLaunch S) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q == 0 && S.kind == NRTGPU_SORT_COLUMN) *S.missing_code = sort_code_of(S.distinct, S.n_distinct, S.missing_value);
  if (q >= S.nq || !S.queries[q].has_after) return;
  const int64_t local = (int64_t)S.after_docs[q] - S.doc_base;
  uint64_t key;
  if (S.kind == NRTGPU_SORT_DOCID && S.reverse) {
    key = local < 0 ? 0ull : (local >= S.n_docs ? 0xffffffffffffffffull : ((uint64_t)((uint32_t)local + 1u) << 32));
  } else {
    uint32_t code = 0; bool exact = true, missing_follow = false;
    if (S.kind == NRTGPU_SORT_COLUMN) {
      const int64_t v = S.after_values[q];
      code = sort_code_of(S.distinct, S.n_distinct, v);
      exact = (code & 1u) == 0u || v == S.missing_value;
      missing_follow = !exact && code == sort_code_of(S.distinct, S.n_distinct, S.missing_value) &&
                       (S.reverse ? S.missing_value < v : S.missing_value > v);
    }
    const uint32_t hi = sort_hi(S.kind, S.reverse, code, 0);
    if (missing_follow) key = ((uint64_t)hi + 1ull) << 32;                  // every doc with this code lacks a value and follows
    else if (!exact) key = (uint64_t)hi << 32;                              // no doc with this code follows: the doc part is moot
    else if (local < 0) key = ((uint64_t)hi + 1ull) << 32;                  // every tied doc here follows afterDoc
    else if (local >= S.n_docs) key = (uint64_t)hi << 32;                   // every tied doc here precedes it
    else key = ((uint64_t)hi << 32) | (uint32_t)(~(uint32_t)local);
  }
  S.queries[q].after_key = key;
}

// FieldDoc.fields[0] of the final hits
struct SortValuesLaunch {
  const int32_t* docs; const int32_t* counts; int32_t nq, top_k, doc_base, kind;
  const int64_t* c64; const int32_t* c32; const uint8_t* has; int64_t missing_value;
  int64_t* out_values; float* out_scores;
};
__global__ void sort_values_kernel(SortValuesLaunch S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S.nq * S.top_k) return;
  const int q = i / S.top_k, r = i % S.top_k;
  if (S.out_scores) S.out_scores[i] = __int_as_float(0x7fc00000);   // NaN: TopFieldCollector does not track scores
  if (r >= S.counts[q]) { S.out_values[i] = 0; return; }
  const int32_t g = S.docs[i], d = g - S.doc_base;
  if (S.kind == NRTGPU_SORT_DOCID) { S.out_values[i] = g; return; }
  if (S.has && !S.has[d]) { S.out_values[i] = S.missing_value; return; }
  S.out_values[i] = S.c32 ? (int64_t)S.c32[d] : S.c64[d];
}

// index time: codes + sorted distinct values of one column (device pointers; codes zeroed by the caller: 0 = no value)
inline int sort_codes_build(const int64_t* c64, const int32_t* c32, const uint8_t* has, int32_t n, uint32_t* codes,
                            uint64_t* keys_tmp, int32_t* idx_tmp, int32_t* rank_tmp, uint64_t* distinct, int32_t* n_distinct_out) {
  if (n <= 0) { *n_distinct_out = 0; return NRTGPU_OK; }
  // the docs that have a value, then their sortable keys, sorted
  int32_t n_has = n;
  if (has) n_has = (int32_t)(thrust::copy_if(thrust::device, thrust::counting_iterator<int32_t>(0), thrust::counting_iterator<int32_t>(n), has, idx_tmp, SortNonZero()) - idx_tmp);
  else thrust::sequence(thrust::device, idx_tmp, idx_tmp + n);
  if (n_has <= 0) { *n_distinct_out = 0; return NRTGPU_OK; }
  sort_col_keys_kernel<<<(unsigned)((n_has + 255) / 256), 256>>>(c64, c32, idx_tmp, n_has, keys_tmp);
  NRT_CUDA_TRY(cudaGetLastError());
  thrust::sort_by_key(thrust::device, keys_tmp, keys_tmp + n_has, idx_tmp);
  sort_mark_kernel<<<(unsigned)((n_has + 255) / 256), 256>>>(keys_tmp, n_has, rank_tmp);
  NRT_CUDA_TRY(cudaGetLastError());
  thrust::inclusive_scan(thrust::device, rank_tmp, rank_tmp + n_has, rank_tmp);
  sort_scatter_kernel<<<(unsigned)((n_has + 255) / 256), 256>>>(keys_tmp, idx_tmp, rank_tmp, n_has, codes, distinct);
  NRT_CUDA_TRY(cudaGetLastError());
  int32_t last = 0;
  NRT_CUDA_TRY(cudaMemcpy(&last, rank_tmp + n_has - 1, sizeof(int32_t), cudaMemcpyDeviceToHost));
  *n_distinct_out = last;
  return NRTGPU_OK;
}

// ---- sort orders of several fields (nrtgpu_sort_order; Lucene Sort of 1..8 SortFields, TopFieldCollector) ----
// An order ranks every doc of the leaf once: perm (position -> doc) and rank (doc -> position + 1) under the fields that
// follow a leading SCORE, up to and including the first DOCID (fields after a DOCID cannot decide anything), then doc id
// asc. The posting kernel keys a hit by its rank: hi = ~rank, lo = ~doc (the COLUMN key with the rank as its code), or,
// for [score, ...], hi = the ordered score, lo = ~rank (kSortScoreRank; the merge decodes the rank as the "doc", and
// sort_fields_values_kernel maps it back through perm). A score, a tie code and a doc would not fit 64 bits together;
// the rank holds the doc tie-break, which is why SCORE must lead. A KEYWORD field is one more key pass
// (sort_order_kw_keys_kernel): the posting kernels read the rank either way, never the field's values.
constexpr int32_t kSortScoreRank = 4;   // internal sort kind of the posting kernels (beside NRTGPU_SORT_COLUMN / _DOCID)
constexpr int kMaxSortFields = 8;

// A KEYWORD field (NRTGPU_SORT_KEYWORD) reads a keyword column's codes (2i + 2 for term i of the image's dictionary, 0: no
// value): `codes` per doc (SORTED), or per value behind the doc offsets `mv_off` (SORTED_SET, ascending within a doc);
// `missing` is 0 (STRING_FIRST) or 1 (STRING_LAST). Its value is the selected code, so values compare as terms only
// between codes of one dictionary.
struct SortFieldDev {
  int32_t kind, reverse, selector, n_distinct;
  int64_t missing;
  const int64_t* c64; const int32_t* c32; const uint8_t* has;
  const int64_t* mv_off;       // multi-valued column: per-doc offsets into c64 (values ascending within a doc)
  const uint32_t* codes;       // single-valued column: order-preserving codes (0 = no value), with its distinct values
  const uint64_t* distinct;
};

// the keyword code of doc d (0: no value): SORTED its code; SORTED_SET the selector's pick of its n ascending codes
// (SortedSetSelector: MIN [0], MAX [n-1], MIDDLE_MIN [(n-1)/2], MIDDLE_MAX [n/2])
__device__ __forceinline__ uint32_t sort_kw_code(const SortFieldDev& f, int32_t d) {
  if (!f.mv_off) return f.codes[d];
  const int64_t a = f.mv_off[d], n = f.mv_off[d + 1] - a;
  if (n == 0) return 0u;
  const int64_t j = f.selector == NRTGPU_SELECT_MAX ? n - 1
                  : f.selector == NRTGPU_SELECT_MIDDLE_MIN ? (n - 1) / 2
                  : f.selector == NRTGPU_SELECT_MIDDLE_MAX ? n / 2 : 0;
  return f.codes[a + j];
}

// the doc's value of one field: the column value (MIN / MAX selected on a multi-valued column) or missing; the global doc
// id; a keyword's selected code
__device__ __forceinline__ int64_t sort_field_value(const SortFieldDev& f, int32_t d, int32_t doc_base) {
  if (f.kind == NRTGPU_SORT_DOCID) return (int64_t)d + doc_base;
  if (f.kind == NRTGPU_SORT_KEYWORD) return (int64_t)sort_kw_code(f, d);
  if (f.mv_off) {
    const int64_t a = f.mv_off[d], b = f.mv_off[d + 1];
    return a == b ? f.missing : f.c64[f.selector == NRTGPU_SELECT_MAX ? b - 1 : a];
  }
  if (f.has && !f.has[d]) return f.missing;
  return f.c32 ? (int64_t)f.c32[d] : f.c64[d];
}
// ascending key of a keyword code: code 0 (no value) first or last by the missing rule, then the whole under reverse
__host__ __device__ __forceinline__ uint64_t sort_kw_key(int32_t reverse, int64_t missing_last, int64_t code) {
  const uint64_t k = code == 0 ? (missing_last ? ~0ull : 0ull) : (uint64_t)code;
  return k ^ (reverse ? ~0ull : 0ull);
}
// ascending key of a value under the field's direction
__device__ __forceinline__ uint64_t sort_field_key(const SortFieldDev& f, int64_t v) {
  if (f.kind == NRTGPU_SORT_KEYWORD) return sort_kw_key(f.reverse, f.missing, v);
  return sortable_u64(v) ^ (f.reverse ? ~0ull : 0ull);
}

// LSD pass keys, in the current perm order: 32-bit codes for single-valued columns, 64-bit keys otherwise
__global__ void sort_order_keys32_kernel(SortFieldDev f, const int32_t* __restrict__ perm, int32_t n, uint32_t* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t c = f.codes[perm[i]];
  if (c == 0u) c = sort_code_of(f.distinct, f.n_distinct, f.missing);
  keys[i] = f.reverse ? ~c : c;
}
// keyword pass: the doc's selected code (codes stay below 2^31 + 2), 0 first or last by the missing rule, under reverse
__global__ void sort_order_kw_keys_kernel(SortFieldDev f, const int32_t* __restrict__ perm, int32_t n, uint32_t* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t c = sort_kw_code(f, perm[i]);
  if (c == 0u) c = f.missing ? 0xffffffffu : 0u;
  keys[i] = f.reverse ? ~c : c;
}
__global__ void sort_order_keys64_kernel(SortFieldDev f, const int32_t* __restrict__ perm, int32_t n, int32_t doc_base,
                                         uint64_t* __restrict__ keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  keys[i] = sort_field_key(f, sort_field_value(f, perm[i], doc_base));
}
__global__ void sort_order_init_kernel(int32_t n, int32_t descending, int32_t* __restrict__ perm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) perm[i] = descending ? n - 1 - i : i;
}
__global__ void sort_order_rank_kernel(const int32_t* __restrict__ perm, int32_t n, uint32_t* __restrict__ rank) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) rank[perm[i]] = (uint32_t)i + 1u;
}

// perm / rank of the fields f[0..n_f) (device pointers; scratch: n keys of each width). Stable LSD sorts on `st`, from the
// last field to the first, starting from doc order (a trailing DOCID sets the start order instead of a pass).
inline int sort_order_build(const SortFieldDev* f, int n_f, int32_t n, int32_t doc_base, cudaStream_t st, int32_t* perm,
                            uint32_t* rank, uint32_t* keys32, uint64_t* keys64) {
  if (n <= 0) return NRTGPU_OK;
  const unsigned grid = (unsigned)((n + 255) / 256);
  const bool docid_last = n_f > 0 && f[n_f - 1].kind == NRTGPU_SORT_DOCID;
  sort_order_init_kernel<<<grid, 256, 0, st>>>(n, docid_last && f[n_f - 1].reverse, perm);
  NRT_CUDA_TRY(cudaGetLastError());
  for (int i = n_f - (docid_last ? 2 : 1); i >= 0; --i) {
    if (f[i].kind == NRTGPU_SORT_KEYWORD || f[i].codes) {
      if (f[i].kind == NRTGPU_SORT_KEYWORD) sort_order_kw_keys_kernel<<<grid, 256, 0, st>>>(f[i], perm, n, keys32);
      else sort_order_keys32_kernel<<<grid, 256, 0, st>>>(f[i], perm, n, keys32);
      NRT_CUDA_TRY(cudaGetLastError());
      thrust::stable_sort_by_key(thrust::cuda::par.on(st), keys32, keys32 + n, perm);
    } else {
      sort_order_keys64_kernel<<<grid, 256, 0, st>>>(f[i], perm, n, doc_base, keys64);
      NRT_CUDA_TRY(cudaGetLastError());
      thrust::stable_sort_by_key(thrust::cuda::par.on(st), keys64, keys64 + n, perm);
    }
  }
  sort_order_rank_kernel<<<grid, 256, 0, st>>>(perm, n, rank);
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

struct SortFieldsAfterLaunch {
  DevQuery* queries; int32_t nq;
  const int32_t* after_docs;      // [nq] global doc ids
  const int64_t* after_values;    // [nq][n_fields]
  int32_t n_fields;               // row length of after_values
  int32_t score_first, score_reverse;
  int32_t n_rank;                 // fields of the rank: f[0..n_rank) = after_values columns score_first .. score_first + n_rank
  SortFieldDev f[kMaxSortFields];
  const int32_t* perm; int32_t n_docs, doc_base;
};

// patches DevQuery::after_key (a hit qualifies iff key < after_key, PagingFieldCollector): pos = the docs of the leaf whose
// (rank fields, global doc) tuple is <= (after values, after_doc), found by a binary search of perm; a doc qualifies on the
// rank iff its rank (1-based) > pos. After values need not be held by any doc; after_doc may lie outside the leaf.
__global__ void sort_fields_after_kernel(SortFieldsAfterLaunch S) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= S.nq || !S.queries[q].has_after) return;
  const int64_t* av = S.after_values + (size_t)q * S.n_fields;
  const int64_t after_doc = S.after_docs[q];
  int lo = 0, hi = S.n_docs;   // first position whose tuple is > the after tuple
  while (lo < hi) {
    const int m = (lo + hi) >> 1;
    const int32_t d = S.perm[m];
    int c = 0;
    for (int i = 0; i < S.n_rank && c == 0; ++i) {
      const uint64_t kd = sort_field_key(S.f[i], sort_field_value(S.f[i], d, S.doc_base));
      const uint64_t ka = sort_field_key(S.f[i], av[S.score_first + i]);
      c = kd < ka ? -1 : (kd > ka ? 1 : 0);
    }
    if (c == 0) c = (int64_t)d + S.doc_base <= after_doc ? -1 : 1;
    if (c < 0) lo = m + 1; else hi = m;
  }
  const uint32_t pos = (uint32_t)lo;
  uint64_t key;
  if (S.score_first) {
    const uint32_t s = float_to_ordered(__uint_as_float((uint32_t)av[0])) ^ (S.score_reverse ? ~0u : 0u);
    key = ((uint64_t)s << 32) | (uint32_t)~pos;
  } else {
    key = (uint64_t)(uint32_t)~pos << 32;
  }
  S.queries[q].after_key = key;
}

// FieldDoc.fields of the final hits ([nq][top_k][n_fields]); score-first orders (and sorted nested top hits, `ranks`): the
// "doc" is a rank + doc_base, mapped back to the doc through perm; the score is recovered from the key's score word
struct SortFieldsValuesLaunch {
  int32_t* docs; const int32_t* counts; int32_t nq, top_k, doc_base, n_fields, score_first, score_reverse, ranks;
  SortFieldDev f[kMaxSortFields];   // every field of the sort (a SCORE entry takes the hit's score)
  const int32_t* perm;
  float* scores; int64_t* out_values;
};
__global__ void sort_fields_values_kernel(SortFieldsValuesLaunch S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S.nq * S.top_k) return;
  const int q = i / S.top_k, r = i % S.top_k;
  int64_t* out = S.out_values + (size_t)i * S.n_fields;
  const float key_score = S.scores[i];
  S.scores[i] = __int_as_float(0x7fc00000);   // NaN: TopFieldCollector does not track scores
  if (r >= S.counts[q]) { for (int j = 0; j < S.n_fields; ++j) out[j] = 0; return; }
  int32_t d = S.docs[i] - S.doc_base;
  float score = 0.0f;
  if (S.score_first || S.ranks) {
    d = S.perm[d - 1];
    S.docs[i] = d + S.doc_base;
  }
  if (S.score_first) score = S.score_reverse ? ordered_to_float(~float_to_ordered(key_score)) : key_score;
  for (int j = 0; j < S.n_fields; ++j)
    out[j] = S.f[j].kind == NRTGPU_SORT_SCORE ? (int64_t)__float_as_uint(score) : sort_field_value(S.f[j], d, S.doc_base);
}

// ---- TopFieldDocs.merge of packed sorted records (nrtgpu_merge_sorted_packed; record layout in include/nrtgpu.h) ----
// Word offsets of the parts of one sorted record: docs [nq*top_k] | counts [nq] | flags [nq] | pad to 8 B | totalHits [nq]
// int64 | values [nq*top_k*n_fields] int64. Every part that holds int64 starts on an even word.
struct SortedRecordLayout {
  int64_t counts, flags, totals, values, words;
};
__host__ __device__ inline SortedRecordLayout sorted_record_layout(int32_t nq, int32_t top_k, int32_t n_fields) {
  SortedRecordLayout L;
  const int64_t n = (int64_t)nq * top_k;
  L.counts = n; L.flags = n + nq;
  L.totals = (n + 2ll * nq + 1) & ~1ll;
  L.values = L.totals + 2ll * nq;
  L.words = L.values + 2 * n * n_fields;
  return L;
}

constexpr int kSortMergeThreads = 256;

struct SortMergeLaunch {
  const int32_t* records;        // [n_lists][L.words]
  int32_t* out;                  // [L.words]
  SortedRecordLayout L;
  int32_t n_lists, nq, top_k, n_fields;
  int32_t n_cmp;                 // fields that decide: up to and including the first DOCID
  int32_t kind[kMaxSortFields], reverse[kMaxSortFields];
  int32_t missing_last;              // bit f: KEYWORD field f is STRING_LAST (else STRING_FIRST)
};

// entries of query q in record r (clamped to [0, top_k])
__device__ __forceinline__ int sort_record_count(const int32_t* r, int64_t counts, int q, int K) {
  const int c = r[counts + q];
  return c < 0 ? 0 : (c > K ? K : c);
}

// ascending merge key of one FieldDoc value: COLUMN / DOCID by the sortable long, SCORE by its float bits, higher first,
// KEYWORD by its code under the missing rule (codes of one dictionary: the records' producer maps them there)
__device__ __forceinline__ uint64_t sort_merge_key(int32_t kind, int32_t reverse, int64_t missing, int64_t v) {
  if (kind == NRTGPU_SORT_SCORE) {
    const uint32_t o = float_to_ordered(__uint_as_float((uint32_t)v));
    return (uint64_t)(reverse ? o : ~o);
  }
  if (kind == NRTGPU_SORT_KEYWORD) return sort_kw_key(reverse, missing, v);
  return sortable_u64(v) ^ (reverse ? ~0ull : 0ull);
}

// One CTA per query, a merge by rank: entry i of list l lands at position i + (entries of every other list m that sort
// before it), each counted by a binary search of list m. Entries that tie on every field and the doc are ordered by list
// (lists m < l first), so the positions are a permutation even then; global doc ids of distinct leaves never tie.
// An entry stops searching once its position reaches top_k. Slots past the merged count are zeroed.
__global__ void __launch_bounds__(kSortMergeThreads) sort_merge_kernel(SortMergeLaunch S) {
  const int q = blockIdx.x;
  const int tid = threadIdx.x;
  const SortedRecordLayout L = S.L;
  const int K = S.top_k, F = S.n_fields;
  int32_t* out_docs = S.out + (size_t)q * K;
  int64_t* out_vals = (int64_t*)(S.out + L.values) + (size_t)q * K * F;
  __shared__ int32_t s_total;
  if (tid == 0) {
    long long t = 0; int32_t f = 0, n = 0;
    for (int m = 0; m < S.n_lists; ++m) {
      const int32_t* r = S.records + (size_t)m * L.words;
      t += ((const long long*)(r + L.totals))[q];
      f |= r[L.flags + q];
      n += sort_record_count(r, L.counts, q, K);
    }
    n = n < K ? n : K;
    S.out[L.counts + q] = n; S.out[L.flags + q] = f; ((long long*)(S.out + L.totals))[q] = t;
    s_total = n;
  }
  __syncthreads();
  const int n_out = s_total;
  for (int i = n_out + tid; i < K; i += kSortMergeThreads) {
    out_docs[i] = 0;
    for (int j = 0; j < F; ++j) out_vals[(size_t)i * F + j] = 0;
  }
  for (int l = 0; l < S.n_lists; ++l) {
    const int32_t* rl = S.records + (size_t)l * L.words;
    const int cl = sort_record_count(rl, L.counts, q, K);
    const int32_t* docs_l = rl + (size_t)q * K;
    const int64_t* vals_l = (const int64_t*)(rl + L.values) + (size_t)q * K * F;
    for (int i = tid; i < cl; i += kSortMergeThreads) {
      const int32_t doc = docs_l[i];
      const int64_t* v = vals_l + (size_t)i * F;
      uint64_t ke[kMaxSortFields];
#pragma unroll
      for (int f = 0; f < kMaxSortFields; ++f) ke[f] = f < S.n_cmp ? sort_merge_key(S.kind[f], S.reverse[f], (S.missing_last >> f) & 1, v[f]) : 0ull;
      int pos = i;
      for (int m = 0; m < S.n_lists && pos < K; ++m) {
        if (m == l) continue;
        const int32_t* rm = S.records + (size_t)m * L.words;
        const int32_t* docs_m = rm + (size_t)q * K;
        const int64_t* vals_m = (const int64_t*)(rm + L.values) + (size_t)q * K * F;
        int lo = 0, hi = sort_record_count(rm, L.counts, q, K);   // first entry of list m that does not sort before (l, i)
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          const int64_t* w = vals_m + (size_t)mid * F;
          int c = 0;
#pragma unroll
          for (int f = 0; f < kMaxSortFields; ++f) {
            if (f < S.n_cmp && c == 0) {
              const uint64_t k = sort_merge_key(S.kind[f], S.reverse[f], (S.missing_last >> f) & 1, w[f]);
              c = k < ke[f] ? -1 : (k > ke[f] ? 1 : 0);
            }
          }
          if (c == 0) { const int32_t d = docs_m[mid]; c = d < doc ? -1 : (d > doc ? 1 : (m < l ? -1 : 1)); }
          if (c < 0) lo = mid + 1; else hi = mid;
        }
        pos += lo;
      }
      if (pos < K) {
        out_docs[pos] = doc;
        for (int j = 0; j < F; ++j) out_vals[(size_t)pos * F + j] = v[j];
      }
    }
  }
}

// Over several leaves: the KEYWORD FieldDoc values of a leaf's hits, codes of the leaf's dictionary, become codes of the
// reader-wide union before the leaves' records merge. map[j]: field j's leaf -> union ordinal map (NULL: not a keyword,
// or the leaf's dictionary is the union). values [n][n_fields]; 0 (no value, or a slot past the count) stays 0.
struct SortKwMapLaunch {
  int64_t* values; int64_t n; int32_t n_fields;
  const uint32_t* map[kMaxSortFields];
};
__global__ void sort_kw_map_kernel(SortKwMapLaunch S) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S.n) return;
  int64_t* v = S.values + i * S.n_fields;
#pragma unroll
  for (int j = 0; j < kMaxSortFields; ++j)   // (unrolled: map[] stays in parameter space)
    if (j < S.n_fields && S.map[j] && v[j] != 0) v[j] = 2 * (int64_t)S.map[j][v[j] / 2 - 1] + 2;
}

// positions [start_hit, start_hit + w) of each list of a merged sorted record ([n][top_k], the leaves' sorted nested top
// hits of one pass-2 group, list g = (query q_lo + g / size, slot g % size)) -> the caller's layout [nq][size][w]: docs,
// FieldDoc values, NaN scores (TopHitsCollectorManager.reduce: Hit.score = Double.NaN) and the counts past start_hit
struct SortedHitsOutLaunch {
  const int32_t* record; SortedRecordLayout L;
  int32_t n, top_k, n_fields, start_hit, w, q_lo, size;
  int32_t* out_docs; float* out_scores; int32_t* out_counts; int64_t* out_values;
};
__global__ void sorted_hits_out_kernel(SortedHitsOutLaunch S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S.n * S.w) return;
  const int g = i / S.w, r = i % S.w, p = S.start_hit + r;
  const int cnt = S.record[S.L.counts + g];
  const size_t qs = (size_t)(S.q_lo + g / S.size) * S.size + g % S.size;
  const bool hit = p < cnt;
  S.out_docs[qs * S.w + r] = hit ? S.record[(size_t)g * S.top_k + p] : 0;
  S.out_scores[qs * S.w + r] = __int_as_float(0x7fc00000);
  const int64_t* v = (const int64_t*)(S.record + S.L.values) + ((size_t)g * S.top_k + p) * S.n_fields;
  for (int j = 0; j < S.n_fields; ++j) S.out_values[(qs * S.w + r) * S.n_fields + j] = hit ? v[j] : 0;
  if (r == 0) S.out_counts[qs] = max(0, cnt - S.start_hit);
}

// a leaf's sorted or score record after its run: a timed-out query is partial (hit_timeout, relation GTE), and the
// totalHits of a query that terminateAfter cut short are capped at terminateAfterMaxRecallCount (as batch_fetch_impl does
// for host results)
__global__ void record_limits_kernel(int32_t nq, const int32_t* __restrict__ timed_out, long long max_recall,
                                     int32_t* __restrict__ flags, long long* __restrict__ totals) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nq) return;
  if (timed_out && timed_out[q]) flags[q] |= 1 | 4;
  if (max_recall > 0 && (flags[q] & 2) && totals[q] > max_recall) totals[q] = max_recall;
}

}  // namespace nrtgpu
