// Test-only launcher of the kNN candidate-stage kernels (tests/knn_harness.py loads it with ctypes). It launches the
// product kernels themselves, with operands prepared the way nrtgpu_index_build and knn_search_host prepare them, so
// that a test can compare the raw candidate scores and the fused epilogue's survivors with a plain reference.
// Not part of the public ABI (include/nrtgpu.h).
#include <cstdio>
#include <string>
#include "../../nrtsearch_b200/csrc/knn_kernel.cuh"

namespace nrtgpu {
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
}  // namespace nrtgpu
using namespace nrtgpu;

namespace {
// device buffers of one call, freed on every return path
struct Bufs {
  void* p[16] = {};
  int n = 0;
  ~Bufs() { for (int i = 0; i < n; ++i) cudaFree(p[i]); }
  template <class T> int alloc(T** out, size_t count) {
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
#define KH_TRY(expr) do { int rc_ = (expr); if (rc_) return rc_; } while (0)
#define KH_FAIL(msg) do { set_error(msg); return NRTGPU_ERR_INVALID; } while (0)
}  // namespace

#define KH_API extern "C" __attribute__((visibility("default")))

KH_API const char* kh_last_error() { return g_last_error.c_str(); }

// bf16 rounding of the product (tc::f32_to_bf16_kernel), as raw 16-bit patterns
KH_API int kh_f32_to_bf16(const float* in, uint16_t* out, int64_t n) {
  Bufs b;
  float* d_in; __nv_bfloat16* d_out;
  KH_TRY(b.upload(&d_in, in, (size_t)n));
  KH_TRY(b.alloc(&d_out, (size_t)n));
  tc::f32_to_bf16_kernel<<<256, 256>>>(d_in, d_out, (size_t)n);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaMemcpy(out, d_out, (size_t)n * 2, cudaMemcpyDeviceToHost));
  return 0;
}

// tc::knn_gemm_bf16_kernel over corpus rows [n_base, n_base + N) of D[n_total][K] against Q[M][K].
//   S != NULL (unfused): S[M][N] receives the approximate scores.
//   S == NULL (fused):   theta[M] is each query's threshold; filter (per doc, n_docs bytes), live_bits (per doc) and
//                        vec_docs (per ordinal, n_total) are optional; cc[M][cc_cap] receives the survivor keys and
//                        cc_cnt[M] their count (which may exceed cc_cap).
KH_API int kh_gemm_bf16(const float* Q, int M, const float* D, int n_total, int K, int n_base, int N, int sim, float* S,
                        const float* theta, const uint8_t* filter, int n_docs, const uint32_t* live_bits,
                        const int32_t* vec_docs, int cc_cap, uint64_t* cc, int32_t* cc_cnt) {
  if (M <= 0 || N <= 0 || K <= 0 || K % 8 || K > 4096 || n_base < 0 || n_base + N > n_total) KH_FAIL("kh_gemm_bf16: bad shape");
  if (!S && (!theta || !cc || !cc_cnt || cc_cap <= 0)) KH_FAIL("kh_gemm_bf16: fused mode needs theta, cc, cc_cnt");
  Bufs b;
  float *dQ, *dD, *dn2, *dS = nullptr, *dTheta = nullptr;
  float2* dab;
  __nv_bfloat16 *dQb, *dDb;
  KH_TRY(b.upload(&dQ, Q, (size_t)M * K));
  KH_TRY(b.upload(&dD, D, (size_t)n_total * K));
  KH_TRY(b.alloc(&dQb, (size_t)M * K));
  KH_TRY(b.alloc(&dDb, (size_t)n_total * K));
  KH_TRY(b.alloc(&dn2, (size_t)n_total));
  KH_TRY(b.alloc(&dab, (size_t)n_total));
  // corpus side as nrtgpu_index_build prepares it, query side as knn_search_host does
  KH_TRY(knn_prepare_norms(dD, n_total, K, dn2));
  tc::f32_to_bf16_kernel<<<1024, 256>>>(dD, dDb, (size_t)n_total * K);
  knn_ab_kernel<<<(n_total + 255) / 256, 256>>>(dn2, n_total, sim, dab);
  tc::f32_to_bf16_kernel<<<256, 256>>>(dQ, dQb, (size_t)M * K);
  NRT_CUDA_TRY(cudaGetLastError());
  CUtensorMap tmQ, tmD;
  KH_TRY(tc::make_tensor_map_bf16(&tmD, dDb, (uint64_t)n_total, (uint64_t)K, tc::BN));
  KH_TRY(tc::make_tensor_map_bf16(&tmQ, dQb, (uint64_t)M, (uint64_t)K, tc::BM));
  tc::GemmParams G;
  G.M = M; G.N = N; G.K = K; G.n_base = n_base; G.dnorm2 = dn2 + n_base; G.ab = dab + n_base; G.sim = sim;
  G.S = nullptr; G.ldS = N;
  G.theta = nullptr; G.cc = nullptr; G.cc_cnt = nullptr; G.cc_cap = cc_cap;
  G.filter = nullptr; G.vec_docs = nullptr; G.live_bits = nullptr;
  uint64_t* dCC = nullptr; int* dCCn = nullptr;
  if (S) {
    KH_TRY(b.alloc(&dS, (size_t)M * N));
    G.S = dS;
  } else {
    uint8_t* dF = nullptr; uint32_t* dL = nullptr; int32_t* dV = nullptr;
    KH_TRY(b.upload(&dTheta, theta, (size_t)M));
    KH_TRY(b.alloc(&dCC, (size_t)M * cc_cap));
    KH_TRY(b.alloc(&dCCn, (size_t)M));
    NRT_CUDA_TRY(cudaMemset(dCC, 0, (size_t)M * cc_cap * sizeof(uint64_t)));
    NRT_CUDA_TRY(cudaMemset(dCCn, 0, (size_t)M * sizeof(int)));
    if (filter) KH_TRY(b.upload(&dF, filter, (size_t)n_docs));
    if (live_bits) KH_TRY(b.upload(&dL, live_bits, (size_t)(n_docs + 31) / 32));
    if (vec_docs) KH_TRY(b.upload(&dV, vec_docs, (size_t)n_total));
    G.theta = dTheta; G.cc = dCC; G.cc_cnt = dCCn; G.filter = dF; G.live_bits = dL; G.vec_docs = dV;
  }
  NRT_CUDA_TRY(cudaFuncSetAttribute(tc::knn_gemm_bf16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::kGemmSmem));
  const int tiles = ((M + tc::BM - 1) / tc::BM) * ((N + tc::BN - 1) / tc::BN);
  tc::knn_gemm_bf16_kernel<<<tiles, tc::kGemmThreads, tc::kGemmSmem>>>(tmQ, tmD, G);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  if (S) {
    NRT_CUDA_TRY(cudaMemcpy(S, dS, (size_t)M * N * sizeof(float), cudaMemcpyDeviceToHost));
  } else {
    NRT_CUDA_TRY(cudaMemcpy(cc, dCC, (size_t)M * cc_cap * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    NRT_CUDA_TRY(cudaMemcpy(cc_cnt, dCCn, (size_t)M * sizeof(int32_t), cudaMemcpyDeviceToHost));
  }
  return 0;
}

// knn_dot_tile_kernel (the fp32 SIMT candidate stage): S[M][N] for D[N][K] against Q[M][K], any K
KH_API int kh_dot_tile(const float* Q, int M, const float* D, int N, int K, int sim, float* S) {
  if (M <= 0 || N <= 0 || K <= 0 || K > 4096) KH_FAIL("kh_dot_tile: bad shape");
  Bufs b;
  float *dQ, *dD, *dn2, *dS;
  KH_TRY(b.upload(&dQ, Q, (size_t)M * K));
  KH_TRY(b.upload(&dD, D, (size_t)N * K));
  KH_TRY(b.alloc(&dn2, (size_t)N));
  KH_TRY(b.alloc(&dS, (size_t)M * N));
  KH_TRY(knn_prepare_norms(dD, N, K, dn2));
  dim3 grid((N + kKnnTile - 1) / kKnnTile, (M + kKnnTile - 1) / kKnnTile);
  knn_dot_tile_kernel<<<grid, 256>>>(dQ, dD, dn2, M, N, K, sim, dS, N);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  NRT_CUDA_TRY(cudaMemcpy(S, dS, (size_t)M * N * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}
