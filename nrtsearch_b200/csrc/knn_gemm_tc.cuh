// Tensor-core candidate stage of the kNN path: S[q, d] = <Q[q,:], D[d,:]> for a chunk of the corpus, bf16 inputs,
// fp32 accumulation in registers, hand-written for sm_90a:
//   * operands are staged by TMA (cp.async.bulk.tensor.2d, 128-byte swizzle) through a 3-stage mbarrier ring; thread 0
//     refills a stage once all eight warps have released it,
//   * two consumer warpgroups issue wgmma.mma_async m64n128k16 (bf16 -> f32) on shared-memory descriptors, each owning
//     64 query rows of the 128 x 128 output tile,
//   * the epilogue reads the accumulators from registers and applies the similarity's monotone transform (cosine: / |d|,
//     l2: 2 dot - |d|^2): unfused, it stores the approximate scores for the per-query select (knn_select_kernel); fused,
//     it keeps only the values at or above the query's running k'-th best. The exact fp64 re-score (knn_rescore_kernel)
//     restores oracle arithmetic for the surviving candidates, so bf16 only affects which k' = 4k candidates survive.
// Replaces the GEMM-shaped part of ExactVectorQuery's scan
// (reference src/main/java/com/yelp/nrtsearch/server/query/vector/ExactVectorQuery.java:137-173).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include "common.cuh"
#include "../../include/nrtgpu.h"

namespace nrtgpu {
namespace tc {

constexpr int BM = 128, BN = 128, BK = 64, kStages = 3, kWgmmaK = 16;
constexpr int kGemmThreads = 256;   // two consumer warpgroups, 64 query rows each
constexpr int kGemmCtasPerSm = 2;   // two CTAs' shared memory fit one SM: the epilogue of one overlaps the mainloop of the other
constexpr uint32_t kABytes = BM * BK * 2, kBBytes = BN * BK * 2, kStageBytes = kABytes + kBBytes;
// Fused epilogue: a row's survivors of the tile are buffered in shared memory and appended to the query's chunk list with
// ONE global atomicAdd per row (a returning atomic per survivor costs a round trip to L2 each); survivors past kRowCap in
// one tile, rare once the threshold is warm, go out one atomic each.
constexpr int kRowCap = 8;
struct GemmSmemTail {
  uint64_t full[kStages], empty[kStages];
  float2 ab[BN];                 // (a, b) of the tile's vectors
  int cnt[BM];                   // survivors per row of the tile
  uint64_t surv[BM * kRowCap];
};
constexpr size_t kGemmSmem = (size_t)kStages * kStageBytes + sizeof(GemmSmemTail) + 1024 /*alignment slack*/;
static_assert(kGemmCtasPerSm * (kGemmSmem + 1024) <= 233472, "kNN GEMM shared memory exceeds two CTAs per SM");

__device__ __forceinline__ uint32_t s_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(s_u32(b)), "r"(c) : "memory"); }
__device__ __forceinline__ void bar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(s_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(s_u32(b)) : "memory"); }
__device__ __forceinline__ void bar_wait(uint64_t* b, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(s_u32(b)), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int crd0, int crd1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(s_u32(dst)), "l"(map), "r"(s_u32(bar)), "r"(crd0), "r"(crd1) : "memory");
}
// wgmma shared-memory matrix descriptor, K-major, 128-byte swizzle: start >> 4 | LBO 1 (unused for swizzled K-major) |
// SBO 1024 B (8 rows x 128 B) | layout SWIZZLE_128B. The tile bases are 1024-byte aligned, so the base offset is 0.
__device__ __forceinline__ uint64_t make_smem_desc(const void* p) {
  uint64_t d = (uint64_t)((s_u32(p) >> 4) & 0x3fffu);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, both operands K-major bf16 in shared memory, D fp32 in registers
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, "
      "%22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, "
      "%42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, "
      "%62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

struct GemmParams {
  int M, N, K;            // queries, vectors in this chunk, dims
  int n_base;             // ordinal of the chunk's first vector (row coordinate into the corpus tensor map)
  const float* dnorm2;    // chunk-relative |d|^2
  const float2* ab;       // chunk-relative (a, b): approximate score = a * dot + b (cosine: 1/|d|, 0; l2: 2, -|d|^2; else 1, 0)
  int sim;
  float* S; int ldS;      // [M][ldS] approximate scores of the chunk (unfused mode), or NULL
  // fused top-k' epilogue: a value survives if it is >= the query's running k'-th best approximate score
  const float* theta;     // [M]
  uint64_t* cc;           // [M][cc_cap] keys (approx score, ordinal) of this chunk's survivors
  int* cc_cnt;            // [M] (may exceed cc_cap: overflow, detected by the merge kernel)
  int cc_cap;
  const uint8_t* filter;  // per DOC 0/1 or NULL
  const int32_t* vec_docs;  // ordinal -> doc or NULL
  const uint32_t* live_bits;  // liveDocs bitmap or NULL
  // per-query filter rows (KnnQuery.filter): query q keeps doc d iff bit d of row qrow[q] is set; qrow[q] < 0 = no filter
  const uint32_t* qfilter = nullptr;   // [n_rows][qwords]
  const int32_t* qrow = nullptr;       // [M] or NULL
  int qwords = 0;
};

// One 128 x 128 output tile per CTA; grid = query tiles x corpus tiles, query tiles varying fastest so that the CTAs sharing
// a corpus tile run together and the tile is fetched from HBM once and served to the other query tiles by L2.
// kRows: the fused epilogue also applies the per-query filter rows (P.qfilter / P.qrow); a separate instantiation keeps the
// epilogue of unfiltered batches exactly as it was.
template <bool kRows>
__device__ __forceinline__ void knn_gemm_bf16_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& P) {
  extern __shared__ uint8_t gemm_raw[];
  uint8_t* base = (uint8_t*)(((uintptr_t)gemm_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* smA = base;
  uint8_t* smB = base + (size_t)kStages * kABytes;
  GemmSmemTail& T = *(GemmSmemTail*)(base + (size_t)kStages * kStageBytes);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = warp >> 2;
  const int m_tiles = (P.M + BM - 1) / BM;
  const int m0 = (int)(blockIdx.x % m_tiles) * BM, n0 = (int)(blockIdx.x / m_tiles) * BN;
  const int num_kb = (P.K + BK - 1) / BK;
  const bool fused = P.S == nullptr;

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) { bar_init(&T.full[s], 1); bar_init(&T.empty[s], kGemmThreads / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  if (fused && tid < BN) T.ab[tid] = __ldg(P.ab + min(n0 + tid, P.N - 1));
  if (tid < BM) T.cnt[tid] = 0;
  __syncthreads();
  if (tid == 0) {
    for (int kb = 0; kb < num_kb && kb < kStages; ++kb) {
      bar_expect_tx(&T.full[kb], kStageBytes);
      tma_load_2d(smA + (size_t)kb * kABytes, &tmA, &T.full[kb], kb * BK, m0);
      tma_load_2d(smB + (size_t)kb * kBBytes, &tmB, &T.full[kb], kb * BK, P.n_base + n0);
    }
  }

  float d[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) d[i] = 0.0f;
  for (int kb = 0; kb < num_kb; ++kb) {
    const int s = kb % kStages;
    bar_wait(&T.full[s], (kb / kStages) & 1);
    const uint64_t da = make_smem_desc(smA + (size_t)s * kABytes + wg * 64 * 128);   // this warpgroup's 64 query rows
    const uint64_t db = make_smem_desc(smB + (size_t)s * kBBytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / kWgmmaK; ++k)   // advance 16 bf16 = 32 B inside the 128 B swizzle atom: +2 in the address field
      wgmma_m64n128k16(d, da + (uint64_t)(2 * k), db + (uint64_t)(2 * k), (uint32_t)((kb | k) != 0));
    wgmma_commit();
    wgmma_wait<1>();   // the MMAs of k-block kb - 1 have retired: its stage can be refilled
    if (kb > 0) {
      const int ps = (kb - 1) % kStages;
      if (lane == 0) bar_arrive(&T.empty[ps]);
      if (tid == 0 && kb - 1 + kStages < num_kb) {
        const int nk = kb - 1 + kStages;
        bar_wait(&T.empty[ps], ((kb - 1) / kStages) & 1);
        bar_expect_tx(&T.full[ps], kStageBytes);
        tma_load_2d(smA + (size_t)ps * kABytes, &tmA, &T.full[ps], nk * BK, m0);
        tma_load_2d(smB + (size_t)ps * kBBytes, &tmB, &T.full[ps], nk * BK, P.n_base + n0);
      }
      __syncwarp();
    }
  }
  wgmma_wait<0>();

  // accumulator layout of m64nNk16: d[4 j + 2 i + e] is row 16 (warp % 4) + lane / 4 + 8 i, column 8 j + 2 (lane % 4) + e
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = row0 + 8 * i, gq = m0 + row;
    if (gq >= P.M) continue;
    if (!fused) {   // unfused: store the approximate scores
      float* out = P.S + (size_t)gq * P.ldS + n0;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + c0 + e, gd = n0 + c;
          if (gd < P.N) {
            float x = d[4 * j + 2 * i + e];
            if (P.sim == NRTGPU_SIM_COSINE) x = x * rsqrtf(fmaxf(P.dnorm2[gd], 1e-30f));
            else if (P.sim == NRTGPU_SIM_L2) x = 2.0f * x - P.dnorm2[gd];
            out[c] = x;
          }
        }
    } else {        // fused top-k': keep only values that can still enter the query's best k'
      const float th = P.theta[gq];
      const uint32_t* qf = nullptr;   // read once per accumulator row
      if constexpr (kRows) { const int qr = P.qrow[gq]; if (qr >= 0) qf = P.qfilter + (size_t)qr * P.qwords; }
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + c0 + e, gd = n0 + c;
          const float2 ab = T.ab[c];
          const float x = fmaf(ab.x, d[4 * j + 2 * i + e], ab.y);
          if (gd < P.N && x >= th) {
            const int ord = P.n_base + gd;
            bool ok = true;
            if (P.filter || P.live_bits || (kRows && qf)) {
              const int doc = P.vec_docs ? P.vec_docs[ord] : ord;
              if (P.filter) ok = P.filter[doc] != 0;
              if (ok && P.live_bits) ok = (P.live_bits[doc >> 5] >> (doc & 31)) & 1u;
              if (kRows && ok && qf) ok = (qf[doc >> 5] >> (doc & 31)) & 1u;
            }
            if (ok) {
              const uint64_t key = make_key(x, ord);
              const int pos = atomicAdd(&T.cnt[row], 1);
              if (pos < kRowCap) {
                T.surv[row * kRowCap + pos] = key;
              } else {
                const int gp = atomicAdd(P.cc_cnt + gq, 1);
                if (gp < P.cc_cap) P.cc[(size_t)gq * P.cc_cap + gp] = key;
              }
            }
          }
        }
    }
  }
  if (fused) {   // one append per row of the tile
    __syncthreads();
    const int gq = m0 + tid;
    if (tid < BM && gq < P.M) {
      const int n = min(T.cnt[tid], kRowCap);
      if (n > 0) {
        const int pos = atomicAdd(P.cc_cnt + gq, n);
        for (int i = 0; i < n; ++i)
          if (pos + i < P.cc_cap) P.cc[(size_t)gq * P.cc_cap + pos + i] = T.surv[tid * kRowCap + i];
      }
    }
  }
}

__global__ void __launch_bounds__(kGemmThreads, kGemmCtasPerSm)
knn_gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmParams P) {
  knn_gemm_bf16_body<false>(tmA, tmB, P);
}
// the same with per-query filter rows
__global__ void __launch_bounds__(kGemmThreads, kGemmCtasPerSm)
knn_gemm_bf16_rows_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmParams P) {
  knn_gemm_bf16_body<true>(tmA, tmB, P);
}

__global__ void f32_to_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) out[i] = __float2bfloat16_rn(in[i]);
}

// 2-D row-major bf16 tensor map [rows][cols], box = box_rows x 64 columns, 128-byte swizzle
inline int make_tensor_map_bf16(CUtensorMap* map, const void* gptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || !p) {
      set_error("cuTensorMapEncodeTiled is not available from the driver");
      return NRTGPU_ERR_CUDA;
    }
    fn = (EncodeFn)p;
  }
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {cols * 2};
  const cuuint32_t box[2] = {(cuuint32_t)BK, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(gptr), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")"); return NRTGPU_ERR_CUDA; }
  return NRTGPU_OK;
}

}  // namespace tc
}  // namespace nrtgpu
