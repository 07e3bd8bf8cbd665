// Hybrid-search stages on the device: weighted RRF blend and QueryRescore.combine, one CTA per query.
//   blend:   reference .../search/multiretriever/blender/operation/WeightedRrfBlenderOperation.java:52-78 and
//            .../blender/score/WeightedRRFScoreDoc.java:60-77 -- first hit score = boost/(k+rank) (float division),
//            later retrievers add boost/(k+rank) in float in declaration order; the reference's final heap orders by
//            score only (BlenderOperation.java:99-132, ties unordered); ties break on doc asc here.
//   rescore: Lucene QueryRescorer.rescore driven by reference src/main/java/com/yelp/nrtsearch/server/rescore/QueryRescore.java:39-57
//            -- combine = (float)(qw*first + rw*second) in double (or (float)(qw*first) when the second pass does not match),
//            then re-sort (score desc, doc asc).
#pragma once
#include "common.cuh"

namespace nrtgpu {

constexpr int kHybThreads = 256;
constexpr int kHybCap = 4096;

struct RrfLaunch {
  const int32_t* docs;    // [R][nq][top_in]
  const int32_t* counts;  // [R][nq]
  const float* boosts;    // [R]
  const float* scores;    // [R][nq][top_in] retriever scores (score-order blending) or NULL
  int32_t mode;           // 0: weighted RRF; 1 / 2 / 3: WeightedScoreDoc.ScoreMode MAX / SUM / AVG of score * boost
                          // (reference .../blender/score/WeightedScoreDoc.java:57-77, float ops in retriever order)
  int32_t R, nq, top_in, rank_constant, top_out;
  int32_t* out_docs; float* out_scores; int32_t* out_counts; int32_t* out_total;
};

__global__ void __launch_bounds__(kHybThreads) rrf_blend_kernel(RrfLaunch P) {
  __shared__ uint64_t keys[kHybCap];
  __shared__ int n_heads;
  const int q = blockIdx.x, tid = threadIdx.x;
  // gather: key = ~(doc << 32 | r << 16 | rank0) so that the descending sort yields (doc asc, r asc)
  int n = 0;
  for (int r = 0; r < P.R; ++r) {
    const int c = P.counts[(size_t)r * P.nq + q];
    for (int i = tid; i < c; i += kHybThreads) {
      const int32_t d = P.docs[((size_t)r * P.nq + q) * P.top_in + i];
      keys[n + i] = ~(((uint64_t)(uint32_t)d << 32) | ((uint64_t)r << 16) | (uint64_t)i);
    }
    n += c;
  }
  if (tid == 0) n_heads = 0;
  const int m = next_pow2(n < 2 ? 2 : n);
  for (int i = n + tid; i < m; i += kHybThreads) keys[i] = 0ull;
  __syncthreads();
  block_bitonic_sort_desc(keys, m);
  // heads accumulate their group in retriever order, then become (score, doc) keys; the rest become 0
  uint64_t mine[kHybCap / kHybThreads];
  int nm = 0;
  for (int i = tid; i < m; i += kHybThreads) {
    uint64_t out = 0ull;
    if (i < n) {
      const uint64_t k = ~keys[i];
      const uint32_t d = (uint32_t)(k >> 32);
      const bool head = (i == 0) || ((uint32_t)((~keys[i - 1]) >> 32) != d);
      if (head) {
        auto contrib = [&](uint64_t kk) {
          const int r = (int)((kk >> 16) & 0xffff), rank0 = (int)(kk & 0xffff);
          if (P.mode == 0) return __fdiv_rn(P.boosts[r], (float)(P.rank_constant + rank0 + 1));
          return __fmul_rn(P.scores[((size_t)r * P.nq + q) * P.top_in + rank0], P.boosts[r]);
        };
        float s = contrib(k);
        int have = 1;
        for (int j = i + 1; j < n; ++j) {
          const uint64_t kj = ~keys[j];
          if ((uint32_t)(kj >> 32) != d) break;
          const float w = contrib(kj);
          if (P.mode == 0 || P.mode == 2) s = __fadd_rn(s, w);
          else if (P.mode == 1) s = fmaxf(s, w);
          else s = __fdiv_rn(__fadd_rn(__fmul_rn(s, (float)have), w), (float)(have + 1));
          ++have;
        }
        out = make_key(s, (int32_t)d);
        atomicAdd(&n_heads, 1);
      }
    }
    mine[nm++] = out;
  }
  __syncthreads();
  nm = 0;
  for (int i = tid; i < m; i += kHybThreads) keys[i] = mine[nm++];
  __syncthreads();
  block_bitonic_sort_desc(keys, m);
  const int total = n_heads;
  const int keep = total < P.top_out ? total : P.top_out;
  for (int i = tid; i < P.top_out; i += kHybThreads) {   // slots past the count: doc 0, score 0.0 (include/nrtgpu.h)
    const uint64_t k = keys[i < keep ? i : 0];
    P.out_docs[(size_t)q * P.top_out + i] = i < keep ? key_doc(k) : 0;
    P.out_scores[(size_t)q * P.top_out + i] = i < keep ? key_score(k) : 0.0f;
  }
  if (tid == 0) { P.out_counts[q] = keep; P.out_total[q] = total; }
}

struct RescoreLaunch {
  int32_t nq, n_hits;
  const int32_t* counts;   // [nq] or NULL (= n_hits)
  int32_t* docs; float* scores;            // [nq][n_hits] in/out
  const uint8_t* second_matches; const float* second_scores;
  double query_weight, rescore_weight;
};

__global__ void __launch_bounds__(kHybThreads) rescore_combine_kernel(RescoreLaunch P) {
  __shared__ uint64_t keys[kHybCap];
  const int q = blockIdx.x, tid = threadIdx.x;
  const int n = P.counts ? P.counts[q] : P.n_hits;
  const size_t base = (size_t)q * P.n_hits;
  for (int i = tid; i < n; i += kHybThreads) {
    const double first = (double)P.scores[base + i];
    const float s = P.second_matches[base + i]
                        ? (float)(__dadd_rn(__dmul_rn(P.query_weight, first), __dmul_rn(P.rescore_weight, (double)P.second_scores[base + i])))
                        : (float)__dmul_rn(P.query_weight, first);
    keys[i] = make_key(s, P.docs[base + i]);
  }
  const int m = next_pow2(n < 2 ? 2 : n);
  for (int i = n + tid; i < m; i += kHybThreads) keys[i] = 0ull;
  __syncthreads();
  block_bitonic_sort_desc(keys, m);
  for (int i = tid; i < n; i += kHybThreads) {
    P.docs[base + i] = key_doc(keys[i]);
    P.scores[base + i] = key_score(keys[i]);
  }
}

}  // namespace nrtgpu
