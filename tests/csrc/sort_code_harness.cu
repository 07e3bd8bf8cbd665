// Test-only launcher of the index-time sort codes (tests/sort_code_harness.py loads it with ctypes). sh_codes runs
// sort_codes_build, the routine nrtgpu_index_build runs once per single-valued column, on host arrays given by the test;
// sh_code_of runs sort_code_of, the lookup of sort_after_kernel and the multi-field order keys, on a list of probe values.
// So a test can compare the codes, the distinct values and the code of any value with a plain reference. Every entry point
// checks its arguments before it launches: a call that could index a kernel out of bounds answers NRTGPU_ERR_INVALID.
// Not part of the public ABI (include/nrtgpu.h).
#include <string>
#include "../../nrtsearch_b200/csrc/sort_kernel.cuh"

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
using namespace nrtgpu;

namespace {
// device buffers of one call, freed on every return path
struct Bufs {
  void* p[8] = {};
  int n = 0;
  ~Bufs() { for (int i = 0; i < n; ++i) cudaFree(p[i]); }
  template <class T> int alloc(T** out, size_t count) {
    if (n == 8) { set_error("harness: too many buffers"); return NRTGPU_ERR_INVALID; }
    void* q = nullptr;
    NRT_CUDA_TRY(cudaMalloc(&q, count ? count * sizeof(T) : 1));
    p[n++] = q;
    *out = (T*)q;
    return 0;
  }
  template <class T> int upload(T** out, const T* host, size_t count) {
    int rc = alloc(out, count);
    if (rc) return rc;
    NRT_CUDA_TRY(cudaMemcpy(*out, host, count * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
  }
};
#define SH_TRY(expr) do { int rc_ = (expr); if (rc_) return rc_; } while (0)
#define SH_FAIL(msg) do { set_error(msg); return NRTGPU_ERR_INVALID; } while (0)

__global__ void code_of_kernel(const uint64_t* __restrict__ distinct, int32_t n_distinct, const int64_t* __restrict__ probes,
                               int32_t n, uint32_t* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = sort_code_of(distinct, n_distinct, probes[i]);
}
}  // namespace

#define SH_API extern "C" __attribute__((visibility("default")))

SH_API const char* sh_last_error() { return g_last_error.c_str(); }

// sort_codes_build over one column of n docs: exactly one of v64 / v32 holds the values, has (may be NULL) marks the docs
// that have one. Out: codes[n] (0 for a doc without a value), distinct[n] (the first *n_distinct are written, ascending in
// the sortable domain) and *n_distinct.
SH_API int sh_codes(const int64_t* v64, const int32_t* v32, const uint8_t* has, int32_t n, uint32_t* codes, uint64_t* distinct,
                    int32_t* n_distinct) {
  if (n < 0 || !codes || !n_distinct || (n > 0 && !distinct)) SH_FAIL("sh_codes: bad shape");
  if (n > 0 && (v64 == nullptr) == (v32 == nullptr)) SH_FAIL("sh_codes: exactly one of v64 / v32 must be given");
  Bufs b;
  int64_t* d64 = nullptr; int32_t* d32 = nullptr; uint8_t* dHas = nullptr;
  uint32_t* dCodes; uint64_t *dKeys, *dDistinct; int32_t *dIdx, *dRank;
  if (v64) SH_TRY(b.upload(&d64, v64, (size_t)n));
  if (v32) SH_TRY(b.upload(&d32, v32, (size_t)n));
  if (has) SH_TRY(b.upload(&dHas, has, (size_t)n));
  SH_TRY(b.alloc(&dCodes, (size_t)n));
  SH_TRY(b.alloc(&dKeys, (size_t)n));
  SH_TRY(b.alloc(&dIdx, (size_t)n));
  SH_TRY(b.alloc(&dRank, (size_t)n));
  SH_TRY(b.alloc(&dDistinct, (size_t)n));
  if (n > 0) NRT_CUDA_TRY(cudaMemset(dCodes, 0, (size_t)n * sizeof(uint32_t)));   // as nrtgpu_index_build: 0 = no value
  int32_t nd = 0;
  SH_TRY(sort_codes_build(d64, d32, dHas, n, dCodes, dKeys, dIdx, dRank, dDistinct, &nd));
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  if (n > 0) {
    NRT_CUDA_TRY(cudaMemcpy(codes, dCodes, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    NRT_CUDA_TRY(cudaMemcpy(distinct, dDistinct, (size_t)nd * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  }
  *n_distinct = nd;
  return 0;
}

// sort_code_of of every probe value against distinct[n_distinct] (strictly ascending sortable keys): out[n_probes]
SH_API int sh_code_of(const uint64_t* distinct, int32_t n_distinct, const int64_t* probes, int32_t n_probes, uint32_t* out) {
  if (n_distinct < 0 || n_probes <= 0 || !probes || !out || (n_distinct > 0 && !distinct)) SH_FAIL("sh_code_of: bad shape");
  for (int32_t i = 1; i < n_distinct; ++i) if (distinct[i] <= distinct[i - 1]) SH_FAIL("sh_code_of: distinct values not strictly ascending");
  Bufs b;
  uint64_t* dDistinct; int64_t* dProbes; uint32_t* dOut;
  SH_TRY(b.upload(&dDistinct, distinct, (size_t)n_distinct));
  SH_TRY(b.upload(&dProbes, probes, (size_t)n_probes));
  SH_TRY(b.alloc(&dOut, (size_t)n_probes));
  code_of_kernel<<<(unsigned)((n_probes + 255) / 256), 256>>>(dDistinct, n_distinct, dProbes, n_probes, dOut);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaMemcpy(out, dOut, (size_t)n_probes * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  return 0;
}
