// Test-only launcher of the kNN kernels that run after the candidate GEMM (tests/knn_stage_b.py loads it with ctypes;
// tests/csrc/knn_harness.cu is its twin for the candidate stage). It launches the product kernels themselves, with the
// launch shapes of knn_search_host, knn_exact_host and nrtgpu_index_build, on host arrays given by the test, so that a
// test can compare the candidate lists of the select and merge kernels, the re-score's pages and certificate decisions,
// the exact fallback's chunk lists and the index-time norms with a plain reference. Every entry point checks its
// arguments before it launches: a call that could index a kernel out of bounds answers NRTGPU_ERR_INVALID instead.
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
  void* p[32] = {};
  int n = 0;
  ~Bufs() { for (int i = 0; i < n; ++i) cudaFree(p[i]); }
  template <class T> int alloc(T** out, size_t count) {
    if (n == 32) { set_error("harness: too many buffers"); return NRTGPU_ERR_INVALID; }
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

namespace {
// every doc a kernel would read of the ordinals [o0, o1) lies in [0, n_docs)
bool docs_inside(const int32_t* vec_docs, int o0, int o1, int n_docs) {
  if (!vec_docs) return o1 <= n_docs;
  for (int o = o0; o < o1; ++o) if (vec_docs[o] < 0 || vec_docs[o] >= n_docs) return false;
  return true;
}
bool rows_inside(const int32_t* qrow, int nq, int n_rows) {
  for (int q = 0; qrow && q < nq; ++q) if (qrow[q] < -1 || qrow[q] >= n_rows) return false;
  return true;
}
bool counts_inside(const int32_t* cnt, int nq, int hi) {
  for (int q = 0; q < nq; ++q) if (cnt[q] < 0 || cnt[q] > hi) return false;
  return true;
}
constexpr int kMaxKprime = kKnnCandCap - kKnnSelThreads;
}  // namespace

// knn_select_kernel, one launch: folds the scores S[nq][ldS] of the ordinals [chunk_base, chunk_base + n_chunk) into the
// incoming lists cand[nq][kprime] / cand_cnt[nq] (updated in place). theta_out[nq] is in / out: the kernel writes an
// entry only when the query's list is full. filter (bytes), live_bits and the rows qfilter[n_rows][qwords] are per doc
// (n_docs docs), vec_docs[n_ords] maps ordinals to docs; each may be NULL.
KH_API int kh_select(const float* S, int nq, int ldS, int n_chunk, int chunk_base, int kprime, uint64_t* cand,
                     int32_t* cand_cnt, float* theta_out, const uint8_t* filter, const uint32_t* live_bits, int n_docs,
                     const int32_t* vec_docs, int n_ords, const uint32_t* qfilter, int n_rows, int qwords,
                     const int32_t* qrow) {
  if (!S || !cand || !cand_cnt || !theta_out || nq <= 0 || n_chunk <= 0 || ldS < n_chunk || chunk_base < 0) KH_FAIL("kh_select: bad shape");
  if (kprime < 1 || kprime > kMaxKprime) KH_FAIL("kh_select: kprime outside [1, kKnnCandCap - kKnnSelThreads]");
  if (!counts_inside(cand_cnt, nq, kprime)) KH_FAIL("kh_select: cand_cnt outside [0, kprime]");
  if (vec_docs && n_ords < chunk_base + n_chunk) KH_FAIL("kh_select: vec_docs shorter than the chunk's ordinals");
  if (filter || live_bits || qrow) {
    if (n_docs <= 0 || !docs_inside(vec_docs, chunk_base, chunk_base + n_chunk, n_docs)) KH_FAIL("kh_select: a doc outside n_docs");
    if (qrow && (!qfilter || n_rows <= 0 || (int64_t)qwords * 32 < n_docs || !rows_inside(qrow, nq, n_rows))) KH_FAIL("kh_select: bad filter rows");
  }
  Bufs b;
  float *dS, *dTheta; uint64_t* dC; int32_t* dCn;
  uint8_t* dF = nullptr; uint32_t *dL = nullptr, *dR = nullptr; int32_t *dV = nullptr, *dQr = nullptr;
  KH_TRY(b.upload(&dS, S, (size_t)nq * ldS));
  KH_TRY(b.upload(&dC, cand, (size_t)nq * kprime));
  KH_TRY(b.upload(&dCn, cand_cnt, (size_t)nq));
  KH_TRY(b.upload(&dTheta, theta_out, (size_t)nq));
  if (filter) KH_TRY(b.upload(&dF, filter, (size_t)n_docs));
  if (live_bits) KH_TRY(b.upload(&dL, live_bits, (size_t)(n_docs + 31) / 32));
  if (vec_docs) KH_TRY(b.upload(&dV, vec_docs, (size_t)n_ords));
  if (qrow) { KH_TRY(b.upload(&dR, qfilter, (size_t)n_rows * qwords)); KH_TRY(b.upload(&dQr, qrow, (size_t)nq)); }
  KnnSelectLaunch L; L.S = dS; L.ldS = ldS; L.n_chunk = n_chunk; L.chunk_base = chunk_base; L.filter = dF; L.live_bits = dL;
  L.vec_docs = dV; L.kprime = kprime; L.nq = nq; L.cand = dC; L.cand_cnt = dCn; L.theta_out = dTheta;
  L.qfilter = dR; L.qrow = dQr; L.qwords = qwords;
  knn_select_kernel<<<nq, kKnnSelThreads>>>(L);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  NRT_CUDA_TRY(cudaMemcpy(cand, dC, (size_t)nq * kprime * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(cand_cnt, dCn, (size_t)nq * sizeof(int32_t), cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(theta_out, dTheta, (size_t)nq * sizeof(float), cudaMemcpyDeviceToHost));
  return 0;
}

// knn_merge_chunk_kernel: folds the first min(cc_cnt[q], cc_cap) keys of cc[nq][cc_cap] into cand[nq][kprime]. cand,
// cand_cnt, cc_cnt and theta are in / out; *overflow is 0 unless some cc_cnt[q] exceeded cc_cap.
KH_API int kh_merge_chunk(int nq, int kprime, int cc_cap, uint64_t* cand, int32_t* cand_cnt, const uint64_t* cc,
                          int32_t* cc_cnt, float* theta, int32_t* overflow) {
  if (!cand || !cand_cnt || !cc || !cc_cnt || !theta || !overflow || nq <= 0 || cc_cap <= 0) KH_FAIL("kh_merge_chunk: bad shape");
  if (kprime < 1 || kprime > kMaxKprime || kprime + cc_cap > kKnnCandCap) KH_FAIL("kh_merge_chunk: kprime + cc_cap must fit kKnnCandCap");
  if (!counts_inside(cand_cnt, nq, kprime)) KH_FAIL("kh_merge_chunk: cand_cnt outside [0, kprime]");
  for (int q = 0; q < nq; ++q) if (cc_cnt[q] < 0) KH_FAIL("kh_merge_chunk: negative cc_cnt");
  Bufs b;
  uint64_t *dC, *dCC; int32_t *dCn, *dCCn, *dOvf; float* dTheta;
  KH_TRY(b.upload(&dC, cand, (size_t)nq * kprime));
  KH_TRY(b.upload(&dCn, cand_cnt, (size_t)nq));
  KH_TRY(b.upload(&dCC, cc, (size_t)nq * cc_cap));
  KH_TRY(b.upload(&dCCn, cc_cnt, (size_t)nq));
  KH_TRY(b.upload(&dTheta, theta, (size_t)nq));
  KH_TRY(b.alloc(&dOvf, 1));
  NRT_CUDA_TRY(cudaMemset(dOvf, 0, sizeof(int32_t)));
  KnnMergeChunkLaunch M; M.cc = dCC; M.cc_cnt = dCCn; M.cc_cap = cc_cap; M.cand = dC; M.cand_cnt = dCn; M.kprime = kprime;
  M.theta = dTheta; M.overflow = dOvf;
  knn_merge_chunk_kernel<<<nq, kKnnSelThreads>>>(M);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  NRT_CUDA_TRY(cudaMemcpy(cand, dC, (size_t)nq * kprime * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(cand_cnt, dCn, (size_t)nq * sizeof(int32_t), cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(cc_cnt, dCCn, (size_t)nq * sizeof(int32_t), cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(theta, dTheta, (size_t)nq * sizeof(float), cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(overflow, dOvf, sizeof(int32_t), cudaMemcpyDeviceToHost));
  return 0;
}

// knn_rescore_kernel on candidate lists given by the caller (keys of (approximate score, ordinal), cand[nq][kprime]):
// pages out_docs / out_scores [nq][k], out_counts[nq] and the certificate's decision unsafe[nq]. sim may carry kKnnByteFlag.
KH_API int kh_rescore(const float* Q, int nq, const float* D, int n, int dims, int sim, const uint64_t* cand,
                      const int32_t* cand_cnt, int kprime, int k, const int32_t* vec_docs, int doc_base, const float* boosts,
                      float eps_rel, float dmax, int32_t* out_docs, float* out_scores, int32_t* out_counts, int32_t* unsafe) {
  if (!Q || !D || !cand || !cand_cnt || !out_docs || !out_scores || !out_counts || !unsafe || nq <= 0 || n <= 0 || dims <= 0 || dims > 4096)
    KH_FAIL("kh_rescore: bad shape");
  if (kprime < 1 || kprime > kMaxKprime || k < 1 || k > kprime) KH_FAIL("kh_rescore: need 1 <= k <= kprime <= kKnnCandCap - kKnnSelThreads");
  if (!counts_inside(cand_cnt, nq, kprime)) KH_FAIL("kh_rescore: cand_cnt outside [0, kprime]");
  for (int q = 0; q < nq; ++q)
    for (int i = 0; i < cand_cnt[q]; ++i) {
      const int32_t ord = key_doc(cand[(size_t)q * kprime + i]);
      if (ord < 0 || ord >= n) KH_FAIL("kh_rescore: a candidate ordinal outside the corpus");
    }
  Bufs b;
  float *dQ, *dD, *dB = nullptr, *dOS; uint64_t* dC; int32_t *dCn, *dV = nullptr, *dOD, *dOC, *dU;
  KH_TRY(b.upload(&dQ, Q, (size_t)nq * dims));
  KH_TRY(b.upload(&dD, D, (size_t)n * dims));
  KH_TRY(b.upload(&dC, cand, (size_t)nq * kprime));
  KH_TRY(b.upload(&dCn, cand_cnt, (size_t)nq));
  if (vec_docs) KH_TRY(b.upload(&dV, vec_docs, (size_t)n));
  if (boosts) KH_TRY(b.upload(&dB, boosts, (size_t)nq));
  KH_TRY(b.alloc(&dOD, (size_t)nq * k));
  KH_TRY(b.alloc(&dOS, (size_t)nq * k));
  KH_TRY(b.alloc(&dOC, (size_t)nq));
  KH_TRY(b.alloc(&dU, (size_t)nq));
  NRT_CUDA_TRY(cudaMemset(dOD, 0, (size_t)nq * k * 4));
  NRT_CUDA_TRY(cudaMemset(dOS, 0, (size_t)nq * k * 4));
  NRT_CUDA_TRY(cudaMemset(dU, 0xff, (size_t)nq * 4));   // -1: "not written" is visible
  KnnRescoreLaunch R; R.Q = dQ; R.D = dD; R.dims = dims; R.sim = sim; R.cand = dC; R.cand_cnt = dCn; R.kprime = kprime;
  R.vec_docs = dV; R.doc_base = doc_base; R.boosts = dB; R.k = k; R.out_docs = dOD; R.out_scores = dOS; R.out_counts = dOC;
  R.unsafe = dU; R.eps_rel = eps_rel; R.dmax = dmax;
  knn_rescore_kernel<<<nq, 256>>>(R);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  NRT_CUDA_TRY(cudaMemcpy(out_docs, dOD, (size_t)nq * k * 4, cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(out_scores, dOS, (size_t)nq * k * 4, cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(out_counts, dOC, (size_t)nq * 4, cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(unsafe, dU, (size_t)nq * 4, cudaMemcpyDeviceToHost));
  return 0;
}

// knn_exact_chunk_kernel + merge_slices_kernel as knn_exact_host launches them, for the queries qsel[n_sel] of Q[nq][dims]
// over D[n][dims]. ords == NULL: every vector, n_chunks = ceil(n / 4096). ords != NULL (gather mode): a query with row
// r = qrow[q] >= 0 scores the ord_cnt[r] ordinals ords[ord_begin[r] ..] only, n_chunks = ceil(max ord_cnt / 4096), at
// least 1. Returns the chunk lists keys[n_sel][n_chunks][k], cnt[n_sel][n_chunks] and the merged pages [n_sel][k].
KH_API int kh_exact(const float* Q, int nq, const float* D, int n, int dims, int sim, const int32_t* qsel, int n_sel, int k,
                    int n_chunks, const float* boosts, const uint8_t* filter, const uint32_t* live_bits, int n_docs,
                    const int32_t* vec_docs, int doc_base, const uint32_t* qfilter, int n_rows, int qwords,
                    const int32_t* qrow, const int32_t* ords, int64_t n_ords, const int64_t* ord_begin,
                    const int32_t* ord_cnt, uint64_t* keys, int32_t* cnt, int32_t* out_docs, float* out_scores,
                    int32_t* out_counts) {
  if (!Q || !D || !qsel || !keys || !cnt || !out_docs || !out_scores || !out_counts || nq <= 0 || n <= 0 || dims <= 0 ||
      dims > 4096 || n_sel <= 0 || n_sel > 65535) KH_FAIL("kh_exact: bad shape");
  if (k < 1 || k > 1024) KH_FAIL("kh_exact: k outside [1, 1024]");
  for (int i = 0; i < n_sel; ++i) if (qsel[i] < 0 || qsel[i] >= nq) KH_FAIL("kh_exact: qsel outside the queries");
  if (n_docs <= 0 || !docs_inside(vec_docs, 0, n, n_docs)) KH_FAIL("kh_exact: a doc outside n_docs");
  if (qrow && (!qfilter || n_rows <= 0 || (int64_t)qwords * 32 < n_docs || !rows_inside(qrow, nq, n_rows))) KH_FAIL("kh_exact: bad filter rows");
  int want_chunks = (n + kKnnExactChunk - 1) / kKnnExactChunk;
  if (ords) {
    if (!qrow || !ord_begin || !ord_cnt) KH_FAIL("kh_exact: gather mode needs qrow, ord_begin, ord_cnt");
    int max_cnt = 0;
    for (int r = 0; r < n_rows; ++r) {
      if (ord_cnt[r] < 0 || ord_begin[r] < 0 || ord_begin[r] + ord_cnt[r] > n_ords) KH_FAIL("kh_exact: an ordinal list outside ords");
      max_cnt = std::max(max_cnt, ord_cnt[r]);
    }
    for (int64_t i = 0; i < n_ords; ++i) if (ords[i] < 0 || ords[i] >= n) KH_FAIL("kh_exact: an ordinal outside the corpus");
    bool unfiltered = false;
    for (int i = 0; i < n_sel; ++i) unfiltered |= qrow[qsel[i]] < 0;
    const int list_chunks = std::max(1, (max_cnt + kKnnExactChunk - 1) / kKnnExactChunk);
    want_chunks = unfiltered ? std::max(want_chunks, list_chunks) : list_chunks;
  }
  if (n_chunks != want_chunks) KH_FAIL("kh_exact: n_chunks does not cover the vectors scored");
  Bufs b;
  float *dQ, *dD, *dB = nullptr, *dOS; uint8_t* dF = nullptr; uint32_t *dL = nullptr, *dR = nullptr;
  int32_t *dSel, *dV = nullptr, *dQr = nullptr, *dOrds = nullptr, *dOc = nullptr, *dCnt, *dOD, *dOC; int64_t* dOb = nullptr; uint64_t* dKeys;
  KH_TRY(b.upload(&dQ, Q, (size_t)nq * dims));
  KH_TRY(b.upload(&dD, D, (size_t)n * dims));
  KH_TRY(b.upload(&dSel, qsel, (size_t)n_sel));
  if (boosts) KH_TRY(b.upload(&dB, boosts, (size_t)nq));
  if (filter) KH_TRY(b.upload(&dF, filter, (size_t)n_docs));
  if (live_bits) KH_TRY(b.upload(&dL, live_bits, (size_t)(n_docs + 31) / 32));
  if (vec_docs) KH_TRY(b.upload(&dV, vec_docs, (size_t)n));
  if (qrow) { KH_TRY(b.upload(&dR, qfilter, (size_t)n_rows * qwords)); KH_TRY(b.upload(&dQr, qrow, (size_t)nq)); }
  if (ords) {
    KH_TRY(b.upload(&dOrds, ords, (size_t)n_ords));
    KH_TRY(b.upload(&dOb, ord_begin, (size_t)n_rows));
    KH_TRY(b.upload(&dOc, ord_cnt, (size_t)n_rows));
  }
  const size_t n_lists = (size_t)n_sel * n_chunks;
  KH_TRY(b.alloc(&dKeys, n_lists * k));
  KH_TRY(b.alloc(&dCnt, n_lists));
  KH_TRY(b.alloc(&dOD, (size_t)n_sel * k));
  KH_TRY(b.alloc(&dOS, (size_t)n_sel * k));
  KH_TRY(b.alloc(&dOC, (size_t)n_sel));
  NRT_CUDA_TRY(cudaMemset(dOD, 0, (size_t)n_sel * k * 4));
  NRT_CUDA_TRY(cudaMemset(dOS, 0, (size_t)n_sel * k * 4));
  KnnExactLaunch X; X.Q = dQ; X.D = dD; X.n = n; X.dims = dims; X.sim = sim; X.qsel = dSel; X.boosts = dB; X.filter = dF;
  X.live_bits = dL; X.vec_docs = dV; X.k = k; X.n_chunks = n_chunks; X.keys = dKeys; X.cnt = dCnt;
  X.qfilter = dR; X.qrow = dQr; X.qwords = qwords; X.ords = dOrds; X.ord_begin = dOb; X.ord_cnt = dOc;
  knn_exact_chunk_kernel<<<dim3((unsigned)n_chunks, (unsigned)n_sel), 256>>>(X);
  NRT_CUDA_TRY(cudaGetLastError());
  MergeLaunch M; M.slice_keys = dKeys; M.slice_cnt = dCnt; M.n_lists = n_chunks; M.top_k = k; M.nq = n_sel; M.doc_base = doc_base;
  M.out_docs = dOD; M.out_scores = dOS; M.out_counts = dOC;
  M.total_hits = nullptr; M.pruned = nullptr; M.terminated = nullptr; M.terminate_after = 0; M.out_total = nullptr; M.out_flags = nullptr;
  merge_slices_kernel<<<n_sel, kMergeThreads>>>(M);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  NRT_CUDA_TRY(cudaMemcpy(keys, dKeys, n_lists * k * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(cnt, dCnt, n_lists * sizeof(int32_t), cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(out_docs, dOD, (size_t)n_sel * k * 4, cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(out_scores, dOS, (size_t)n_sel * k * 4, cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(out_counts, dOC, (size_t)n_sel * 4, cudaMemcpyDeviceToHost));
  return 0;
}

// the index-time preparation of a vector field as nrtgpu_index_build runs it: knn_prepare_norms -> norm2[n],
// knn_max_norm2_kernel -> *max_norm2, knn_ab_kernel -> ab[n][2]
KH_API int kh_prepare(const float* D, int n, int dims, int sim, float* norm2, float* max_norm2, float* ab) {
  if (!D || !norm2 || !max_norm2 || !ab || n <= 0 || dims <= 0 || dims > 4096) KH_FAIL("kh_prepare: bad shape");
  Bufs b;
  float *dD, *dn2; unsigned int* dMx; float2* dab;
  KH_TRY(b.upload(&dD, D, (size_t)n * dims));
  KH_TRY(b.alloc(&dn2, (size_t)n));
  KH_TRY(b.alloc(&dMx, 1));
  KH_TRY(b.alloc(&dab, (size_t)n));
  KH_TRY(knn_prepare_norms(dD, n, dims, dn2));
  NRT_CUDA_TRY(cudaMemset(dMx, 0, sizeof(unsigned int)));
  knn_max_norm2_kernel<<<256, 256>>>(dn2, n, dMx);
  NRT_CUDA_TRY(cudaGetLastError());
  knn_ab_kernel<<<(n + 255) / 256, 256>>>(dn2, n, sim, dab);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  NRT_CUDA_TRY(cudaMemcpy(norm2, dn2, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(max_norm2, dMx, sizeof(float), cudaMemcpyDeviceToHost));
  NRT_CUDA_TRY(cudaMemcpy(ab, dab, (size_t)n * sizeof(float2), cudaMemcpyDeviceToHost));
  return 0;
}
