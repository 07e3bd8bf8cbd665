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
