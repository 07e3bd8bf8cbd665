// Shared device/host helpers for the nrtgpu kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include "batch_plan.h"

namespace nrtgpu {

#define NRT_CUDA_TRY(expr)                                                                  \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      ::nrtgpu::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));               \
      return (_e == cudaErrorMemoryAllocation) ? NRTGPU_ERR_OOM : NRTGPU_ERR_CUDA;           \
    }                                                                                        \
  } while (0)

#ifdef __CUDACC__
// BM25 term score exactly as Lucene's BM25Scorer.score (float ops, round-to-nearest, never fused):
//   weight - weight / (1f + freq * cache[norm])
__device__ __forceinline__ float bm25_score(float weight, float freq, float norm_inverse) {
  float x = __fmul_rn(freq, norm_inverse);
  x = __fadd_rn(1.0f, x);
  x = __fdiv_rn(weight, x);
  return __fsub_rn(weight, x);
}

// In-place bitonic sort (descending) of n (power of two) 64-bit keys in shared memory by the whole CTA.
__device__ __forceinline__ void block_bitonic_sort_desc(uint64_t* a, int n) {
  for (int k = 2; k <= n; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < (n >> 1); i += blockDim.x) {
        int lo = ((i & ~(j - 1)) << 1) | (i & (j - 1));
        int hi = lo | j;
        bool desc = ((lo & k) == 0);
        uint64_t x = a[lo], y = a[hi];
        if ((x < y) == desc) { a[lo] = y; a[hi] = x; }
      }
      __syncthreads();
    }
  }
}

__device__ __forceinline__ int next_pow2(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

// Candidate buffer flush of a posting kernel (all threads of the CTA): sorts the count keys of cand (cap entries, a power
// of two), keeps the best top_k and, once it holds top_k, publishes the k-th key minus dec as the query's threshold
// g_theta (atomicMax). The CTA's copy theta is raised to the published threshold.
__device__ __forceinline__ void flush_top_k(uint64_t* cand, int& count, int cap, int top_k, unsigned long long dec,
                                            uint64_t* g_theta, unsigned long long& theta) {
  __syncthreads();
  int n = count;
  if (n > cap) n = cap;
  const int m = next_pow2(n < 2 ? 2 : n);
  for (int i = n + threadIdx.x; i < m; i += blockDim.x) cand[i] = 0ull;
  __syncthreads();
  block_bitonic_sort_desc(cand, m);
  if (threadIdx.x == 0) {
    const int keep = n < top_k ? n : top_k;
    count = keep;
    if (keep == top_k) {
      const unsigned long long kth = cand[top_k - 1] - dec;
      const unsigned long long old = atomicMax((unsigned long long*)g_theta, kth);
      const unsigned long long t = old > kth ? old : kth;
      if (t > theta) theta = t;
    } else {
      const unsigned long long g = *(volatile unsigned long long*)g_theta;
      if (g > theta) theta = g;
    }
  }
  __syncthreads();
}

// Deadline of a run (SearchCutoffWrapper): the first work item of the run stamps *clock0 with %globaltimer; an item
// that starts more than deadline_ns later is late. deadline_ns < 0: the request's budget was spent before the launch.
// Called by one thread per work item, only when a deadline is set (deadline_ns != 0).
__device__ __forceinline__ bool deadline_passed(long long deadline_ns, unsigned long long* clock0) {
  if (deadline_ns < 0) return true;
  unsigned long long now;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
  unsigned long long t0 = atomicCAS(clock0, 0ull, now);
  if (t0 == 0ull) t0 = now;
  return now > t0 && now - t0 > (unsigned long long)deadline_ns;   // (another CTA may have stamped clock0 after this one read the timer)
}
#endif

}  // namespace nrtgpu
