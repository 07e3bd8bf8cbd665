// Exact kNN over an HBM-resident float vector field (ExactVectorQuery semantics,
// reference src/main/java/com/yelp/nrtsearch/server/query/vector/ExactVectorQuery.java:137-173;
// score = VectorSimilarityFunction.compare(q, v) * boost, .../search/KnnUtils.java:62-64).
//
// Two stages per batch:
//   A. candidate generation: tiled fp32 dot products of every (query, vector) pair, streamed in doc
//      chunks; a per-query select keeps the best k' = 2k candidates by the fp32 score;
//   B. exact re-score of the k' candidates with double accumulation (the oracle's arithmetic) and the
//      Lucene score mapping in float, then the final (score desc, doc asc) top-k.
// Stage A is the GEMM-shaped part (the tensor-core version replaces only that stage).
#pragma once
#include <algorithm>
#include <cstring>
#include <vector>
#include "common.cuh"
#include "bool_kernel.cuh"
#include "knn_gemm_tc.cuh"
#include "../../include/nrtgpu.h"

namespace nrtgpu {

constexpr int kKnnTile = 64;       // queries x docs per CTA tile
constexpr int kKnnKStep = 16;
constexpr int kKnnChunk = 32768;   // docs per streamed chunk
constexpr int kKnnSelThreads = 256;
constexpr int kKnnCandCap = 4096;
constexpr int kKnnWarmChunk = 32768;   // vectors scored through the unfused path to seed the thresholds of the fused chunks

// per-vector squared magnitude (double accumulate -> float)
__global__ void knn_norm2_kernel(const float* __restrict__ v, int n, int dims, float* __restrict__ out) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n) return;
  const float* p = v + (size_t)warp * dims;
  double s = 0.0;
  for (int i = lane; i < dims; i += 32) { double x = p[i]; s += x * x; }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) out[warp] = (float)s;
}

__global__ void knn_max_norm2_kernel(const float* __restrict__ norm2, int n, unsigned int* __restrict__ out_bits) {
  float m = 0.0f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = fmaxf(m, norm2[i]);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(out_bits, __float_as_uint(m));   // m >= 0: float order == unsigned order
}

// (a, b) with approximate score = a * dot + b, monotone in the final Lucene score of the similarity
__global__ void knn_ab_kernel(const float* __restrict__ norm2, int n, int sim, float2* __restrict__ ab) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float2 r = make_float2(1.0f, 0.0f);
  if (sim == NRTGPU_SIM_COSINE) r.x = rsqrtf(fmaxf(norm2[i], 1e-30f));
  else if (sim == NRTGPU_SIM_L2) r = make_float2(2.0f, -norm2[i]);
  ab[i] = r;
}

inline int knn_prepare_norms(const float* d_vec, int n, int dims, float* d_out) {
  int threads = 256, warps_per_block = threads / 32;
  knn_norm2_kernel<<<(n + warps_per_block - 1) / warps_per_block, threads>>>(d_vec, n, dims, d_out);
  NRT_CUDA_TRY(cudaGetLastError());
  return NRTGPU_OK;
}

// approximate raw similarity used only to rank candidates (monotone in the final score):
//   dot / cosine / mip: dot (cosine divides by |d|), l2: -(|q|^2 + |d|^2 - 2 dot)
__global__ void __launch_bounds__(256) knn_dot_tile_kernel(const float* __restrict__ Q, const float* __restrict__ D,
                                                           const float* __restrict__ dnorm2, int nq, int n_chunk,
                                                           int dims, int sim, float* __restrict__ S /*[nq][chunk]*/,
                                                           int ldS) {
  __shared__ float sq[kKnnKStep][kKnnTile + 1];
  __shared__ float sd[kKnnKStep][kKnnTile + 1];
  const int tq = threadIdx.x / 16, td = threadIdx.x % 16;  // 16x16 threads, 4x4 outputs each
  const int q0 = blockIdx.y * kKnnTile, d0 = blockIdx.x * kKnnTile;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < dims; k0 += kKnnKStep) {
    for (int i = threadIdx.x; i < kKnnTile * kKnnKStep; i += 256) {
      int r = i / kKnnKStep, c = i % kKnnKStep;
      int k = k0 + c;
      sq[c][r] = (q0 + r < nq && k < dims) ? Q[(size_t)(q0 + r) * dims + k] : 0.0f;
      sd[c][r] = (d0 + r < n_chunk && k < dims) ? D[(size_t)(d0 + r) * dims + k] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kKnnKStep; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = sq[k][tq * 4 + i]; b[i] = sd[k][td * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int q = q0 + tq * 4 + i;
    if (q >= nq) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int d = d0 + td * 4 + j;
      if (d >= n_chunk) continue;
      float v = acc[i][j];
      if (sim == NRTGPU_SIM_COSINE) v = v * rsqrtf(fmaxf(dnorm2[d], 1e-30f));
      else if (sim == NRTGPU_SIM_L2) v = 2.0f * v - dnorm2[d];  // -(d2) + |q|^2 (constant per query)
      S[(size_t)q * ldS + d] = v;
    }
  }
}

// per query: fold one chunk of approximate scores into the running best-k' candidate list
struct KnnSelectLaunch {
  const float* S; int ldS; int n_chunk; int chunk_base;  // ordinal of S[:,0]
  const uint8_t* filter;   // per DOC 0/1 or NULL
  const uint32_t* live_bits;  // liveDocs bitmap or NULL (deleted docs are never hits: IndexSearcher acceptDocs)
  const int32_t* vec_docs; // ord -> doc or NULL
  int kprime; int nq;
  uint64_t* cand;          // [nq][kprime] sorted desc keys (approx score, ord)
  int32_t* cand_cnt;       // [nq]
  float* theta_out;        // optional [nq]: the k'-th best approximate score once the list is full (threshold of the fused chunks)
  // per-query filter rows: query q keeps doc d iff bit d of row qrow[q] is set; qrow[q] < 0 = no filter
  const uint32_t* qfilter = nullptr; const int32_t* qrow = nullptr; int qwords = 0;
};

__global__ void __launch_bounds__(kKnnSelThreads) knn_select_kernel(KnnSelectLaunch L) {
  __shared__ uint64_t buf[kKnnCandCap];
  __shared__ int count;
  __shared__ unsigned long long theta;
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const int qr = L.qrow ? L.qrow[q] : -1;
  const uint32_t* qf = qr >= 0 ? L.qfilter + (size_t)qr * L.qwords : nullptr;
  int have = L.cand_cnt[q];
  for (int i = tid; i < have; i += kKnnSelThreads) buf[i] = L.cand[(size_t)q * L.kprime + i];
  if (tid == 0) { count = have; theta = (have == L.kprime) ? L.cand[(size_t)q * L.kprime + L.kprime - 1] : 0ull; }
  __syncthreads();
  int ub = have;
  auto compact = [&]() {   // returns the number of keys kept (CTA-uniform)
    __syncthreads();
    int n = count;
    int m = next_pow2(n < 2 ? 2 : n);
    for (int i = n + tid; i < m; i += kKnnSelThreads) buf[i] = 0ull;
    __syncthreads();
    block_bitonic_sort_desc(buf, m);
    const int keep = n < L.kprime ? n : L.kprime;
    if (tid == 0) { count = keep; if (keep == L.kprime) theta = buf[L.kprime - 1]; }
    __syncthreads();
    return keep;
  };
  for (int i0 = 0; i0 < L.n_chunk; i0 += kKnnSelThreads) {
    int i = i0 + tid;
    bool is_cand = false; uint64_t key = 0;
    if (i < L.n_chunk) {
      int ord = L.chunk_base + i;
      bool ok = true;
      if (L.filter || L.live_bits || qf) {
        const int doc = L.vec_docs ? L.vec_docs[ord] : ord;
        if (L.filter) ok = L.filter[doc] != 0;
        if (ok && L.live_bits) ok = (L.live_bits[doc >> 5] >> (doc & 31)) & 1u;
        if (ok && qf) ok = (qf[doc >> 5] >> (doc & 31)) & 1u;
      }
      if (ok) { key = make_key(L.S[(size_t)q * L.ldS + i], ord); is_cand = key > theta; }
    }
    unsigned bal = __ballot_sync(0xffffffffu, is_cand);
    if (bal) {
      int base = 0;
      if (lane == 0) base = atomicAdd(&count, __popc(bal));
      base = __shfl_sync(0xffffffffu, base, 0);
      if (is_cand) buf[base + __popc(bal & ((1u << lane) - 1))] = key;
    }
    ub += kKnnSelThreads;
    if (ub > kKnnCandCap - kKnnSelThreads) {
      __syncthreads();
      const int seen = count;
      __syncthreads();   // every thread has read the count before anybody appends again
      ub = (seen > kKnnCandCap - kKnnSelThreads) ? compact() : seen;
    }
  }
  const int keep = compact();
  for (int i = tid; i < keep; i += kKnnSelThreads) L.cand[(size_t)q * L.kprime + i] = buf[i];
  if (tid == 0) {
    L.cand_cnt[q] = keep;
    if (L.theta_out && keep == L.kprime) L.theta_out[q] = key_score(buf[L.kprime - 1]);
  }
}

// exact re-score (double accumulation, Lucene score mapping in float) + final top-k; one CTA per query
struct KnnRescoreLaunch {
  const float* Q; const float* D; int dims; int sim;
  const uint64_t* cand; const int32_t* cand_cnt; int kprime;
  const int32_t* vec_docs; int doc_base; const float* boosts; int k;
  int32_t* out_docs; float* out_scores; int32_t* out_counts;
  // rank-safety certificate of the candidate stage: unsafe[q] = 1 unless every vector OUTSIDE the candidate list is
  // proven to score below the k-th exact score. eps_rel bounds the relative error of the candidate stage's dot product
  // in units of |q||d| (bf16 operands: 2^-7; fp32 SIMT: dims * 2^-23), dmax = largest |d| in the corpus.
  int32_t* unsafe; float eps_rel; float dmax;
};

// VectorSimilarityFunction.compare -> score, float vectors (VectorFieldDef.java:664-673) and byte vectors (:870-881: the same
// except DOT_PRODUCT = 0.5 + dot / (dims * 2^15)); sim carries kKnnByteFlag for byte vectors
constexpr int kKnnByteFlag = 0x100;
__device__ __forceinline__ float knn_map_score(int sim, int dims, double dot, double na, double nb, double d2) {
  const int base = sim & 0xff;
  float s;
  if (base == NRTGPU_SIM_L2) s = __fdiv_rn(1.0f, __fadd_rn(1.0f, (float)d2));
  else if (base == NRTGPU_SIM_DOT) {
    if (sim & kKnnByteFlag) s = __fadd_rn(0.5f, __fdiv_rn((float)dot, (float)(dims * (1 << 15))));
    else { s = __fdiv_rn(__fadd_rn(1.0f, (float)dot), 2.0f); s = s > 0.f ? s : 0.f; }
  } else if (base == NRTGPU_SIM_COSINE) { const float cs = (float)(dot / sqrt(na * nb)); s = __fdiv_rn(__fadd_rn(1.0f, cs), 2.0f); s = s > 0.f ? s : 0.f; }
  else { const float t = (float)dot; s = t < 0.f ? __fdiv_rn(1.0f, __fadd_rn(1.0f, __fmul_rn(-1.0f, t))) : __fadd_rn(t, 1.0f); }
  return s;
}

// largest final score a vector whose APPROXIMATE score is <= th can have (monotone score mapping applied to th + error bound)
__device__ __forceinline__ float knn_score_upper_bound(int sim_flags, int dims, double th, double qn, double dmax, double eps_rel, float boost) {
  const double slack = 1.0 + 1e-3;   // rsqrt / float norm / accumulation rounding on top of the operand rounding
  const int sim = sim_flags & 0xff;
  double s;
  if (sim == NRTGPU_SIM_DOT && (sim_flags & kKnnByteFlag)) {
    s = 0.5 + (th + eps_rel * slack * qn * dmax) / ((double)dims * 32768.0);
  } else if (sim == NRTGPU_SIM_COSINE) {            // approx = dot / |d|  (|q| cos)
    const double c = (th + eps_rel * slack * qn) / fmax(qn, 1e-300);
    s = (1.0 + fmin(c, 1.0)) / 2.0;
  } else if (sim == NRTGPU_SIM_L2) {         // approx = 2 dot - |d|^2 = |q|^2 - dist^2
    const double d2 = qn * qn - (th + 2.0 * eps_rel * slack * qn * dmax);
    s = 1.0 / (1.0 + fmax(d2, 0.0));
  } else {                                   // approx = dot
    const double d = th + eps_rel * slack * qn * dmax;
    if (sim == NRTGPU_SIM_DOT) s = (1.0 + d) / 2.0;
    else s = d < 0.0 ? 1.0 / (1.0 - d) : d + 1.0;
  }
  if (s < 0.0) s = 0.0;
  float f = (float)(s * (1.0 + 1e-6));
  f = __fmul_ru(f, boost);
  return f;
}

__global__ void __launch_bounds__(256) knn_rescore_kernel(KnnRescoreLaunch L) {
  __shared__ uint64_t keys[kKnnCandCap];
  const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = L.cand_cnt[q];
  const float* qv = L.Q + (size_t)q * L.dims;
  const float boost = L.boosts ? L.boosts[q] : 1.0f;
  __shared__ double q_norm2;
  if (warp == 0) {
    double s = 0.0;
    for (int i = lane; i < L.dims; i += 32) { const double x = qv[i]; s += x * x; }
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) q_norm2 = s;
  }
  for (int c = warp; c < n; c += 8) {
    int ord = key_doc(L.cand[(size_t)q * L.kprime + c]);
    const float* dv = L.D + (size_t)ord * L.dims;
    double dot = 0, na = 0, nb = 0, d2 = 0;
    for (int i = lane; i < L.dims; i += 32) {
      double x = qv[i], y = dv[i];
      dot += x * y; na += x * x; nb += y * y; d2 += (x - y) * (x - y);
    }
    for (int o = 16; o > 0; o >>= 1) {
      dot += __shfl_xor_sync(0xffffffffu, dot, o); na += __shfl_xor_sync(0xffffffffu, na, o);
      nb += __shfl_xor_sync(0xffffffffu, nb, o);  d2 += __shfl_xor_sync(0xffffffffu, d2, o);
    }
    if (lane == 0) {
      // VectorSimilarityFunction.compare (reference VectorFieldDef.java:664-673 restates the mapping)
      float s = knn_map_score(L.sim, L.dims, dot, na, nb, d2);
      s = __fmul_rn(s, boost);
      int doc = L.vec_docs ? L.vec_docs[ord] : ord;
      keys[c] = make_key(s, doc);
    }
  }
  __syncthreads();
  int m = next_pow2(n < 2 ? 2 : n);
  for (int i = n + tid; i < m; i += 256) keys[i] = 0ull;
  __syncthreads();
  block_bitonic_sort_desc(keys, m);
  int keep = n < L.k ? n : L.k;
  for (int i = tid; i < keep; i += 256) {
    L.out_docs[(size_t)q * L.k + i] = key_doc(keys[i]) + L.doc_base;
    L.out_scores[(size_t)q * L.k + i] = key_score(keys[i]);
  }
  if (tid == 0) {
    L.out_counts[q] = keep;
    if (L.unsafe) {
      int bad = 0;
      if (n == L.kprime) {   // the list is full: vectors outside it exist, all with approximate scores <= the weakest candidate's
        const double th = (double)key_score(L.cand[(size_t)q * L.kprime + n - 1]);
        const float ub = knn_score_upper_bound(L.sim, L.dims, th, sqrt(q_norm2), (double)L.dmax, (double)L.eps_rel, boost);
        bad = !(n >= L.k && ub < key_score(keys[L.k - 1]));
      }
      L.unsafe[q] = bad;
    }
  }
}

// Exact fallback of the queries the certificate rejected: every vector of a 4096-vector chunk is scored with the oracle's
// arithmetic (fp64 accumulation, Lucene score mapping in float, x boost), the chunk's best k keys go to a slice list and
// merge_slices_kernel merges the chunks -- ExactVectorQuery.java:137-173 literally.
constexpr int kKnnExactChunk = 4096;
struct KnnExactLaunch {
  const float* Q; const float* D; int n, dims, sim;
  const int32_t* qsel;         // [n_sel] query ordinals
  const float* boosts; const uint8_t* filter; const uint32_t* live_bits; const int32_t* vec_docs;
  int k, n_chunks;
  uint64_t* keys;              // [n_sel][n_chunks][k]
  int32_t* cnt;                // [n_sel][n_chunks]
  // per-query filter rows: query q keeps doc d iff bit d of row qrow[q] is set; qrow[q] < 0 = no filter
  const uint32_t* qfilter = nullptr; const int32_t* qrow = nullptr; int qwords = 0;
  // optional gather mode: a query with filter row r scores only the ord_cnt[r] ordinals ords[ord_begin[r] ..] of its row's
  // docs instead of every vector (chunk c covers list entries [c * kKnnExactChunk, (c + 1) * kKnnExactChunk))
  const int32_t* ords = nullptr; const int64_t* ord_begin = nullptr; const int32_t* ord_cnt = nullptr;
};

__global__ void __launch_bounds__(256) knn_exact_chunk_kernel(KnnExactLaunch L) {
  __shared__ uint64_t keys[kKnnExactChunk];
  const int chunk = blockIdx.x, sel = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int q = L.qsel[sel];
  const float* qv = L.Q + (size_t)q * L.dims;
  const float boost = L.boosts ? L.boosts[q] : 1.0f;
  const int qr = L.qrow ? L.qrow[q] : -1;
  const uint32_t* qf = qr >= 0 ? L.qfilter + (size_t)qr * L.qwords : nullptr;
  const int32_t* list = (L.ords && qr >= 0) ? L.ords + L.ord_begin[qr] : nullptr;
  const int base = chunk * kKnnExactChunk;
  const int m = min(kKnnExactChunk, (list ? L.ord_cnt[qr] : L.n) - base);
  for (int c = warp; c < kKnnExactChunk; c += 8) {
    uint64_t key = 0ull;
    if (c < m) {
      const int ord = list ? list[base + c] : base + c;
      const int doc = L.vec_docs ? L.vec_docs[ord] : ord;
      bool ok = true;
      if (L.filter) ok = L.filter[doc] != 0;
      if (ok && L.live_bits) ok = (L.live_bits[doc >> 5] >> (doc & 31)) & 1u;
      if (ok && qf) ok = (qf[doc >> 5] >> (doc & 31)) & 1u;
      if (ok) {
        const float* dv = L.D + (size_t)ord * L.dims;
        double dot = 0, na = 0, nb = 0, d2 = 0;
        for (int i = lane; i < L.dims; i += 32) {
          const double x = qv[i], y = dv[i];
          dot += x * y; na += x * x; nb += y * y; d2 += (x - y) * (x - y);
        }
        for (int o = 16; o > 0; o >>= 1) {
          dot += __shfl_xor_sync(0xffffffffu, dot, o); na += __shfl_xor_sync(0xffffffffu, na, o);
          nb += __shfl_xor_sync(0xffffffffu, nb, o);  d2 += __shfl_xor_sync(0xffffffffu, d2, o);
        }
        const float s = knn_map_score(L.sim, L.dims, dot, na, nb, d2);
        key = make_key(__fmul_rn(s, boost), doc);
      }
    }
    if (lane == 0) keys[c] = key;
  }
  __syncthreads();
  block_bitonic_sort_desc(keys, kKnnExactChunk);
  int have = 0;   // keys are > 0 for real hits, 0 for filtered / padding
  for (int i = tid; i < L.k; i += 256) {
    const uint64_t kk = keys[i];
    L.keys[((size_t)sel * L.n_chunks + chunk) * L.k + i] = kk;
    if (kk) have = i + 1;
  }
  have = __reduce_max_sync(0xffffffffu, have);
  __shared__ int wmax[8];
  if (lane == 0) wmax[warp] = have;
  __syncthreads();
  if (tid == 0) { int h = 0; for (int w = 0; w < 8; ++w) h = max(h, wmax[w]); L.cnt[(size_t)sel * L.n_chunks + chunk] = h; }
}

// fused path: fold the survivors of one chunk into the running best-k' list and refresh the query's threshold
struct KnnMergeChunkLaunch {
  uint64_t* cc; int* cc_cnt; int cc_cap;
  uint64_t* cand; int32_t* cand_cnt; int kprime;
  float* theta; int* overflow;
};

__global__ void __launch_bounds__(kKnnSelThreads) knn_merge_chunk_kernel(KnnMergeChunkLaunch L) {
  __shared__ uint64_t buf[kKnnCandCap];
  const int q = blockIdx.x, tid = threadIdx.x;
  const int have = L.cand_cnt[q];
  int nc = L.cc_cnt[q];
  if (nc > L.cc_cap) { if (tid == 0) *L.overflow = 1; nc = L.cc_cap; }
  for (int i = tid; i < have; i += kKnnSelThreads) buf[i] = L.cand[(size_t)q * L.kprime + i];
  for (int i = tid; i < nc; i += kKnnSelThreads) buf[have + i] = L.cc[(size_t)q * L.cc_cap + i];
  const int n = have + nc;
  const int m = next_pow2(n < 2 ? 2 : n);
  for (int i = n + tid; i < m; i += kKnnSelThreads) buf[i] = 0ull;
  __syncthreads();
  block_bitonic_sort_desc(buf, m);
  const int keep = n < L.kprime ? n : L.kprime;
  for (int i = tid; i < keep; i += kKnnSelThreads) L.cand[(size_t)q * L.kprime + i] = buf[i];
  if (tid == 0) {
    L.cand_cnt[q] = keep;
    L.cc_cnt[q] = 0;
    if (keep == L.kprime) L.theta[q] = key_score(buf[L.kprime - 1]);
  }
}

__global__ void fill_f32_kernel(float* p, int n, float v) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// Scratch slots of a kNN call: knn_search_host's, then the per-query filters' (nrtgpu.cu). knn_exact_host runs after the
// candidate stage and reuses two: its slice keys take the unfused score matrix's slot, its counts and pages the chunk buffer's.
enum class KnnSlot : int {
  Theta, ChunkCand, ChunkCandCnt, Overflow, Q, Scores, Cand, CandCnt, OutDocs, OutScores, OutCounts, Boosts, Filter, Qbf16,
  Unsafe, ExactSel, Qrow, Rows, TermBits, Terms, RowMeta, GatherQ, GatherBoosts, Ords, OrdBegin, GatherRows, GatherQrow,
  Count, ExactKeys = Scores, ExactCnt = ChunkCand
};

// device scratch of one kNN call: slots grow on demand and are kept between calls (no cudaMalloc / cudaFree, which
// synchronise the device, on the request path). The index owns one and serialises the calls that use it.
struct KnnScratch {
  void* p[(int)KnnSlot::Count] = {};
  size_t cap[(int)KnnSlot::Count] = {};
  ~KnnScratch() { for (auto q : p) if (q) cudaFree(q); }
  int get(int i, size_t bytes, void** out) {
    if (bytes > cap[i]) {
      if (p[i]) { cudaFree(p[i]); p[i] = nullptr; cap[i] = 0; }
      NRT_CUDA_TRY(cudaMalloc(&p[i], bytes));
      cap[i] = bytes;
    }
    *out = p[i];
    return 0;
  }
};
#define NRT_KNN_GET(slot, ptr, bytes) do { int rc_ = sc.get((int)(slot), (bytes), (void**)&(ptr)); if (rc_) return rc_; } while (0)

// what the kNN stages read of an index image (nrtgpu_index::knn_corpus)
struct KnnCorpus {
  const float* vec; const float* norm2; const int32_t* vec_docs;   // [n][dims] vectors, their |v|^2, ordinal -> doc or NULL
  int n, dims, sim, doc_base, n_docs;                              // sim | kKnnByteFlag for byte vectors
  const uint32_t* live_bits; float dmax;                           // liveDocs bitmap or NULL; largest |v|
  // tensor-core candidate stage: bf16 copy of the vectors, its TMA tensor map, per-vector (a, b); NULL: fp32 SIMT stage
  const __nv_bfloat16* bf16 = nullptr; const CUtensorMap* tmap = nullptr; const float2* ab = nullptr;
};

// a batch of queries, in host memory
struct KnnRequest {
  const float* queries; int nq, k;   // [nq][dims]
  const float* boosts; const uint8_t* filter;   // [nq] or NULL; [n_docs] bytes (0 = excluded) or NULL
  // query q keeps doc d iff bit d of row qrow[q] of d_rows (device, [rows][words]) is set; qrow NULL or qrow[q] < 0: no row
  const uint32_t* d_rows; const int32_t* qrow; int words;
};

struct KnnPages { int32_t* docs; float* scores; int32_t* counts; };   // host [nq][k], [nq][k], [nq]

// page i of src -> page sel[i] of dst, for i < n
inline void knn_scatter(const KnnPages& src, int n, const int32_t* sel, const KnnPages& dst, int k) {
  for (int i = 0; i < n; ++i) {
    std::memcpy(dst.docs + (size_t)sel[i] * k, src.docs + (size_t)i * k, (size_t)k * 4);
    std::memcpy(dst.scores + (size_t)sel[i] * k, src.scores + (size_t)i * k, (size_t)k * 4);
    dst.counts[sel[i]] = src.counts[i];
  }
}

// Runs fn(request, pages) on the queries sel[] of req, their vectors, boosts and rows packed into a request of their own,
// and writes its pages to rows sel[i] of out. A selection 0, 1, ..., n - 1 runs on req's own arrays and out, uncopied.
template <class Fn>
int knn_run_subset(const KnnRequest& req, int dims, const std::vector<int32_t>& sel, const KnnPages& out, Fn&& fn) {
  const int n = (int)sel.size(), k = req.k;
  KnnRequest r = req; r.nq = n;
  bool prefix = true;
  for (int i = 0; i < n; ++i) prefix &= sel[(size_t)i] == i;
  if (prefix) return fn(r, out);
  std::vector<float> qv((size_t)n * dims), bv((size_t)n), sv((size_t)n * k);
  std::vector<int32_t> rv((size_t)n), dv((size_t)n * k), cv((size_t)n);
  for (int i = 0; i < n; ++i) {
    const int q = sel[(size_t)i];
    std::memcpy(qv.data() + (size_t)i * dims, req.queries + (size_t)q * dims, (size_t)dims * 4);
    if (req.boosts) bv[(size_t)i] = req.boosts[q];
    if (req.qrow) rv[(size_t)i] = req.qrow[q];
  }
  r.queries = qv.data(); r.boosts = req.boosts ? bv.data() : nullptr; r.qrow = req.qrow ? rv.data() : nullptr;
  const KnnPages packed{dv.data(), sv.data(), cv.data()};
  const int rc = fn(r, packed);
  if (!rc) knn_scatter(packed, n, sel.data(), out, k);
  return rc;
}

// Exact evaluation of the queries sel[] (rows of X.Q) with the oracle's arithmetic over n_chunks chunks of kKnnExactChunk
// vectors each (X.ords set: of their filter row's ordinal list); merge_slices_kernel merges the chunks' lists and the
// pages overwrite rows sel[i] of out. X carries the queries, k and the filters.
inline int knn_exact_host(const KnnCorpus& corpus, KnnScratch& sc, cudaStream_t st, KnnExactLaunch X, int n_chunks,
                          const std::vector<int32_t>& sel, const KnnPages& out) {
  const int n_sel = (int)sel.size(), k = X.k;
  X.D = corpus.vec; X.n = corpus.n; X.dims = corpus.dims; X.sim = corpus.sim; X.live_bits = corpus.live_bits; X.vec_docs = corpus.vec_docs;
  int32_t *dSel = nullptr, *dCnt = nullptr, *dXD = nullptr, *dXC = nullptr; uint64_t* dKeys = nullptr; float* dXS = nullptr;
  NRT_KNN_GET(KnnSlot::ExactSel, dSel, (size_t)n_sel * sizeof(int32_t));
  NRT_CUDA_TRY(cudaMemcpyAsync(dSel, sel.data(), (size_t)n_sel * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  // the slice lists can be large (n_sel * n_chunks * k keys): process the selected queries in groups that fit 256 MB
  // (and the 65535 rows of a grid's y dimension)
  const size_t per_q = (size_t)n_chunks * k * sizeof(uint64_t);
  const int group = (int)std::max<size_t>(1, std::min<size_t>({(size_t)n_sel, ((size_t)256 << 20) / per_q, (size_t)65535}));
  NRT_KNN_GET(KnnSlot::ExactKeys, dKeys, (size_t)group * per_q);
  NRT_KNN_GET(KnnSlot::ExactCnt, dCnt, (size_t)group * n_chunks * sizeof(int32_t) + (size_t)group * k * 8 + (size_t)group * 4);
  dXD = dCnt + (size_t)group * n_chunks; dXS = (float*)(dXD + (size_t)group * k); dXC = (int32_t*)(dXS + (size_t)group * k);
  std::vector<int32_t> hd((size_t)group * k), hc((size_t)group); std::vector<float> hs((size_t)group * k);
  for (int g0 = 0; g0 < n_sel; g0 += group) {
    const int gn = std::min(group, n_sel - g0);
    X.qsel = dSel + g0; X.n_chunks = n_chunks; X.keys = dKeys; X.cnt = dCnt;
    knn_exact_chunk_kernel<<<dim3((unsigned)n_chunks, (unsigned)gn), 256, 0, st>>>(X);
    NRT_CUDA_TRY(cudaGetLastError());
    MergeLaunch M; M.slice_keys = dKeys; M.slice_cnt = dCnt; M.n_lists = n_chunks; M.top_k = k; M.nq = gn; M.doc_base = corpus.doc_base;
    M.out_docs = dXD; M.out_scores = dXS; M.out_counts = dXC;
    M.total_hits = nullptr; M.pruned = nullptr; M.terminated = nullptr; M.terminate_after = 0; M.out_total = nullptr; M.out_flags = nullptr;
    merge_slices_kernel<<<gn, kMergeThreads, 0, st>>>(M);
    NRT_CUDA_TRY(cudaGetLastError());
    NRT_CUDA_TRY(cudaMemcpyAsync(hd.data(), dXD, (size_t)gn * k * 4, cudaMemcpyDeviceToHost, st));
    NRT_CUDA_TRY(cudaMemcpyAsync(hs.data(), dXS, (size_t)gn * k * 4, cudaMemcpyDeviceToHost, st));
    NRT_CUDA_TRY(cudaMemcpyAsync(hc.data(), dXC, (size_t)gn * 4, cudaMemcpyDeviceToHost, st));
    NRT_CUDA_TRY(cudaStreamSynchronize(st));
    knn_scatter(KnnPages{hd.data(), hs.data(), hc.data()}, gn, sel.data() + g0, out, k);
  }
  return NRTGPU_OK;
}

// The top-k pages of req over the corpus. stage_ms (optional): [0] = candidate GEMM kernels, [1] = select kernels, [2] =
// exact re-score (CUDA events on st). n_uncertified (optional): the queries that took the exact fallback.
inline int knn_search_host(const KnnCorpus& corpus, const KnnRequest& req, KnnScratch& sc, cudaStream_t st,
                           const KnnPages& out, float* stage_ms, int32_t* n_uncertified) {
  const int n = corpus.n, dims = corpus.dims, sim = corpus.sim, nq = req.nq, k = req.k;
  const bool use_tc = corpus.bf16 != nullptr && corpus.tmap != nullptr && corpus.ab != nullptr;
  int kprime = use_tc ? (4 * k < 128 ? 128 : 4 * k) : (2 * k < 64 ? 64 : 2 * k);
  if (kprime > kKnnCandCap - kKnnSelThreads) kprime = kKnnCandCap - kKnnSelThreads;
  bool fused = use_tc && kprime <= 1024;           // best-k' (<= 1024) + chunk survivors (<= 3072) fit one 4096-key sort
  const int cc_cap = kKnnCandCap - 1024;
  float *dQ = nullptr, *dS = nullptr, *dB = nullptr, *dOS = nullptr, *dTheta = nullptr; uint8_t* dF = nullptr;
  uint64_t *dC = nullptr, *dCC = nullptr; __nv_bfloat16* dQb = nullptr;
  int32_t *dCn = nullptr, *dOD = nullptr, *dOC = nullptr, *dQrow = nullptr, *dUnsafe = nullptr, *dCCn = nullptr, *dOvf = nullptr;
  const int chunk_max = use_tc ? 65536 : kKnnChunk;
  if (fused) {
    NRT_KNN_GET(KnnSlot::Theta, dTheta, (size_t)nq * sizeof(float));
    NRT_KNN_GET(KnnSlot::ChunkCand, dCC, (size_t)nq * cc_cap * sizeof(uint64_t));
    NRT_KNN_GET(KnnSlot::ChunkCandCnt, dCCn, (size_t)nq * sizeof(int));
    NRT_KNN_GET(KnnSlot::Overflow, dOvf, sizeof(int));
    NRT_CUDA_TRY(cudaMemsetAsync(dCCn, 0, (size_t)nq * sizeof(int), st));
    NRT_CUDA_TRY(cudaMemsetAsync(dOvf, 0, sizeof(int), st));
    fill_f32_kernel<<<(nq + 255) / 256, 256, 0, st>>>(dTheta, nq, -INFINITY);
  }
  int chunk = n < chunk_max ? n : chunk_max;
  chunk = (chunk + 3) & ~3;   // keep score rows 16-byte aligned
  NRT_KNN_GET(KnnSlot::Q, dQ, (size_t)nq * dims * sizeof(float));
  // fused mode: the first kKnnWarmChunk vectors go through the UNFUSED path (scores stored, knn_select_kernel) to seed
  // every query's threshold; with an empty threshold the fused epilogue would have to keep every value it sees
  const int warm = fused ? (n < kKnnWarmChunk ? ((n + 3) & ~3) : kKnnWarmChunk) : 0;
  NRT_KNN_GET(KnnSlot::Scores, dS, (size_t)nq * (fused ? warm : chunk) * sizeof(float));
  NRT_KNN_GET(KnnSlot::Cand, dC, (size_t)nq * kprime * sizeof(uint64_t));
  NRT_KNN_GET(KnnSlot::CandCnt, dCn, (size_t)nq * sizeof(int32_t));
  NRT_KNN_GET(KnnSlot::OutDocs, dOD, (size_t)nq * k * sizeof(int32_t));
  NRT_KNN_GET(KnnSlot::OutScores, dOS, (size_t)nq * k * sizeof(float));
  NRT_KNN_GET(KnnSlot::OutCounts, dOC, (size_t)nq * sizeof(int32_t));
  if (req.boosts) { NRT_KNN_GET(KnnSlot::Boosts, dB, (size_t)nq * sizeof(float));
                    NRT_CUDA_TRY(cudaMemcpyAsync(dB, req.boosts, (size_t)nq * sizeof(float), cudaMemcpyHostToDevice, st)); }
  if (req.filter) { NRT_KNN_GET(KnnSlot::Filter, dF, (size_t)corpus.n_docs);
                    NRT_CUDA_TRY(cudaMemcpyAsync(dF, req.filter, (size_t)corpus.n_docs, cudaMemcpyHostToDevice, st)); }
  if (req.qrow) { NRT_KNN_GET(KnnSlot::Qrow, dQrow, (size_t)nq * sizeof(int32_t));
                  NRT_CUDA_TRY(cudaMemcpyAsync(dQrow, req.qrow, (size_t)nq * sizeof(int32_t), cudaMemcpyHostToDevice, st)); }
  NRT_CUDA_TRY(cudaMemcpyAsync(dQ, req.queries, (size_t)nq * dims * sizeof(float), cudaMemcpyHostToDevice, st));
  NRT_CUDA_TRY(cudaMemsetAsync(dCn, 0, (size_t)nq * sizeof(int32_t), st));
  CUtensorMap tmQ;
  if (use_tc) {
    NRT_KNN_GET(KnnSlot::Qbf16, dQb, (size_t)nq * dims * sizeof(__nv_bfloat16));
    tc::f32_to_bf16_kernel<<<256, 256, 0, st>>>(dQ, dQb, (size_t)nq * dims);
    NRT_CUDA_TRY(cudaGetLastError());
    if (int rc = tc::make_tensor_map_bf16(&tmQ, dQb, (uint64_t)nq, (uint64_t)dims, tc::BM)) return rc;
  }
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  float gemm_ms = 0.f, select_ms = 0.f;
  if (stage_ms) for (auto& e : ev) NRT_CUDA_TRY(cudaEventCreate(&e));
  // fused mode: warm-up chunk (unfused), then chunks of 64K, 128K, 256K, 256K, ...: with s vectors seen the expected survivors
  // of a chunk of c vectors are k' * c / s per query (800, 533, 457, 213, ... at k' = 400), well inside the chunk buffer (cc_cap)
  int cur = fused ? warm : chunk, n_done = 0;
  for (int base = 0; base < n; base += cur, ++n_done) {
    if (fused && n_done >= 1) cur = n_done == 1 ? 65536 : (n_done == 2 ? 131072 : 262144);
    int nc = n - base < cur ? n - base : cur;
    const bool warm_chunk = fused && n_done == 0;
    if (stage_ms) NRT_CUDA_TRY(cudaEventRecord(ev[0], st));
    if (use_tc) {
      tc::GemmParams G; G.M = nq; G.N = nc; G.K = dims; G.n_base = base; G.dnorm2 = corpus.norm2 + base; G.ab = corpus.ab + base; G.sim = sim & 0xff;
      G.S = (fused && !warm_chunk) ? nullptr : dS; G.ldS = fused ? warm : chunk;
      G.theta = dTheta; G.cc = dCC; G.cc_cnt = dCCn; G.cc_cap = cc_cap; G.filter = dF; G.vec_docs = corpus.vec_docs; G.live_bits = corpus.live_bits;
      G.qfilter = req.d_rows; G.qrow = dQrow; G.qwords = req.words;
      const int tiles = ((nq + tc::BM - 1) / tc::BM) * ((nc + tc::BN - 1) / tc::BN);
      if (dQrow) tc::knn_gemm_bf16_rows_kernel<<<tiles, tc::kGemmThreads, tc::kGemmSmem, st>>>(tmQ, *corpus.tmap, G);
      else tc::knn_gemm_bf16_kernel<<<tiles, tc::kGemmThreads, tc::kGemmSmem, st>>>(tmQ, *corpus.tmap, G);
    } else {
      dim3 grid((nc + kKnnTile - 1) / kKnnTile, (nq + kKnnTile - 1) / kKnnTile);
      knn_dot_tile_kernel<<<grid, 256, 0, st>>>(dQ, corpus.vec + (size_t)base * dims, corpus.norm2 + base, nq, nc, dims, sim & 0xff, dS, chunk);
    }
    NRT_CUDA_TRY(cudaGetLastError());
    if (stage_ms) NRT_CUDA_TRY(cudaEventRecord(ev[1], st));
    if (fused && !warm_chunk) {
      KnnMergeChunkLaunch Mg; Mg.cc = dCC; Mg.cc_cnt = dCCn; Mg.cc_cap = cc_cap; Mg.cand = dC; Mg.cand_cnt = dCn; Mg.kprime = kprime;
      Mg.theta = dTheta; Mg.overflow = dOvf;
      knn_merge_chunk_kernel<<<nq, kKnnSelThreads, 0, st>>>(Mg);
    } else {
      KnnSelectLaunch S; S.S = dS; S.ldS = fused ? warm : chunk; S.n_chunk = nc; S.theta_out = fused ? dTheta : nullptr; S.chunk_base = base; S.filter = dF;
      S.live_bits = corpus.live_bits; S.vec_docs = corpus.vec_docs; S.kprime = kprime; S.nq = nq; S.cand = dC; S.cand_cnt = dCn;
      S.qfilter = req.d_rows; S.qrow = dQrow; S.qwords = req.words;
      knn_select_kernel<<<nq, kKnnSelThreads, 0, st>>>(S);
    }
    NRT_CUDA_TRY(cudaGetLastError());
    if (stage_ms) {
      NRT_CUDA_TRY(cudaEventRecord(ev[2], st));
      NRT_CUDA_TRY(cudaEventSynchronize(ev[2]));
      float a = 0.f, b = 0.f;
      cudaEventElapsedTime(&a, ev[0], ev[1]); cudaEventElapsedTime(&b, ev[1], ev[2]);
      gemm_ms += a; select_ms += b;
    }
  }
  if (fused) {   // a chunk produced more survivors than the buffer holds (adversarial order): redo with the SIMT stage
    int ovf = 0;
    NRT_CUDA_TRY(cudaMemcpyAsync(&ovf, dOvf, sizeof(int), cudaMemcpyDeviceToHost, st));
    NRT_CUDA_TRY(cudaStreamSynchronize(st));
    if (ovf) {
      if (stage_ms) for (auto& e : ev) cudaEventDestroy(e);
      KnnCorpus simt = corpus; simt.bf16 = nullptr; simt.tmap = nullptr; simt.ab = nullptr;
      return knn_search_host(simt, req, sc, st, out, stage_ms, n_uncertified);
    }
  }
  if (stage_ms) NRT_CUDA_TRY(cudaEventRecord(ev[0], st));
  KnnRescoreLaunch R; R.Q = dQ; R.D = corpus.vec; R.dims = dims; R.sim = sim; R.cand = dC; R.cand_cnt = dCn; R.kprime = kprime;
  R.vec_docs = corpus.vec_docs; R.doc_base = corpus.doc_base; R.boosts = dB; R.k = k; R.out_docs = dOD; R.out_scores = dOS; R.out_counts = dOC;
  NRT_KNN_GET(KnnSlot::Unsafe, dUnsafe, (size_t)nq * sizeof(int32_t));
  R.unsafe = dUnsafe; R.dmax = corpus.dmax;
  // bf16 operands: 2^-7 |q||d|; fp32 FMA chain (and byte vectors, whose elements and products are exact in bf16 / fp32): dims * 2^-23
  R.eps_rel = (use_tc && !(sim & kKnnByteFlag)) ? 0.0078125f : (float)dims * 1.1920929e-7f;
  knn_rescore_kernel<<<nq, 256, 0, st>>>(R);
  NRT_CUDA_TRY(cudaGetLastError());
  if (stage_ms) {
    NRT_CUDA_TRY(cudaEventRecord(ev[1], st));
    NRT_CUDA_TRY(cudaEventSynchronize(ev[1]));
    float c = 0.f; cudaEventElapsedTime(&c, ev[0], ev[1]);
    stage_ms[0] = gemm_ms; stage_ms[1] = select_ms; stage_ms[2] = c;
    for (auto& e : ev) cudaEventDestroy(e);
  }
  NRT_CUDA_TRY(cudaMemcpyAsync(out.docs, dOD, (size_t)nq * k * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(out.scores, dOS, (size_t)nq * k * sizeof(float), cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaMemcpyAsync(out.counts, dOC, (size_t)nq * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  std::vector<int32_t> unsafe((size_t)nq);
  NRT_CUDA_TRY(cudaMemcpyAsync(unsafe.data(), dUnsafe, (size_t)nq * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  NRT_CUDA_TRY(cudaStreamSynchronize(st));
  // ---- queries whose candidate list is not certified rank-safe (score clusters tighter than the candidate stage's
  //      error bound, e.g. near-duplicate vectors): exact evaluation of every vector, as ExactVectorQuery does
  std::vector<int32_t> sel;
  for (int q = 0; q < nq; ++q) if (unsafe[(size_t)q]) sel.push_back(q);
  if (n_uncertified) *n_uncertified = (int32_t)sel.size();
  if (!sel.empty()) {
    KnnExactLaunch X; X.Q = dQ; X.boosts = dB; X.filter = dF; X.k = k; X.qfilter = req.d_rows; X.qrow = dQrow; X.qwords = req.words;
    return knn_exact_host(corpus, sc, st, X, (n + kKnnExactChunk - 1) / kKnnExactChunk, sel, out);
  }
  return NRTGPU_OK;
}

}  // namespace nrtgpu
