// Test-only launcher of the relevance top-k kernels (tests/topk_harness.py loads it with ctypes). th_merge_slices runs
// merge_slices_kernel, the per-query merge of one batch's work-item lists, on host arrays with every optional input of
// MergeLaunch; th_flush_top_k runs flush_top_k, the candidate-buffer cut and threshold publication of the posting kernels,
// in one CTA. So a test can compare both with a plain reference at the shapes the engine's searches rarely reach. Every
// entry point checks its arguments before it launches and answers NRTGPU_ERR_INVALID for anything a producer in the engine
// cannot hand the kernels. Not part of the public ABI (include/nrtgpu.h).
#include <string>
#include "../../nrtsearch_b200/csrc/bool_kernel.cuh"

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
    if (n == 16) { set_error("harness: too many buffers"); return NRTGPU_ERR_INVALID; }
    void* q = nullptr;
    NRT_CUDA_TRY(cudaMalloc(&q, count ? count * sizeof(T) : 1));
    p[n++] = q;
    *out = (T*)q;
    return 0;
  }
  // a device copy of host[count], or NULL for a NULL host array
  template <class T> int upload(T** out, const T* host, size_t count) {
    *out = nullptr;
    if (!host) return 0;
    int rc = alloc(out, count);
    if (rc) return rc;
    NRT_CUDA_TRY(cudaMemcpy(*out, host, count * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
  }
  template <class T> static int download(T* host, const T* dev, size_t count) {
    if (host) NRT_CUDA_TRY(cudaMemcpy(host, dev, count * sizeof(T), cudaMemcpyDeviceToHost));
    return 0;
  }
};
#define TH_TRY(expr) do { int rc_ = (expr); if (rc_) return rc_; } while (0)
#define TH_FAIL(msg) do { set_error(msg); return NRTGPU_ERR_INVALID; } while (0)

// a real key encodes a local doc in [0, INT32_MAX - doc_base] (key_doc) and is never 0, the kernels' padding
bool key_ok(uint64_t k, int32_t doc_base) {
  const int32_t d = key_doc(k);
  return k != 0ull && d >= 0 && d <= INT32_MAX - doc_base;
}

// flush_top_k on cand[cap] in dynamic shared memory, as a posting kernel's CTA holds its candidate buffer
__global__ void flush_kernel(uint64_t* g_cand, int32_t cap, int32_t* g_count, int32_t top_k, unsigned long long dec,
                             uint64_t* g_theta, unsigned long long* g_cta_theta) {
  extern __shared__ uint64_t cand[];
  __shared__ int count;
  __shared__ unsigned long long theta;
  for (int i = threadIdx.x; i < cap; i += blockDim.x) cand[i] = g_cand[i];
  if (threadIdx.x == 0) { count = *g_count; theta = *g_cta_theta; }
  flush_top_k(cand, count, cap, top_k, dec, g_theta, theta);
  for (int i = threadIdx.x; i < cap; i += blockDim.x) g_cand[i] = cand[i];
  if (threadIdx.x == 0) { *g_count = count; *g_cta_theta = theta; }
}
}  // namespace

#define TH_API extern "C" __attribute__((visibility("default")))

TH_API const char* th_last_error() { return g_last_error.c_str(); }

// merge_slices_kernel over nq queries of n_lists lists: slice_keys[nq][n_lists][top_k] (list (q, l) holds
// slice_cnt[q][n_lists] keys), one CTA per query. Optional (NULL: absent, as in MergeLaunch): theta[nq], total_hits[nq],
// pruned[nq], terminated[nq] (in/out), known_hits[nq], out_total[nq], out_flags[nq]. The outputs out_docs[nq][top_k],
// out_scores[nq][top_k], out_counts[nq], out_total and out_flags are in/out: their contents are uploaded before the launch,
// so a test sees every slot the kernel leaves unwritten.
TH_API int th_merge_slices(int32_t nq, int32_t n_lists, int32_t top_k, int32_t doc_base, const uint64_t* slice_keys,
                           const int32_t* slice_cnt, const uint64_t* theta, const unsigned long long* total_hits,
                           const int32_t* pruned, int32_t* terminated, long long terminate_after,
                           const unsigned long long* known_hits, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                           long long* out_total, int32_t* out_flags) {
  if (nq <= 0 || n_lists < 0 || top_k <= 0 || top_k > kMaxTopK || doc_base < 0) TH_FAIL("th_merge_slices: bad shape");
  if (!slice_keys || !slice_cnt || !out_docs || !out_scores || !out_counts) TH_FAIL("th_merge_slices: NULL array");
  for (int64_t i = 0; i < (int64_t)nq * n_lists; ++i) {
    const int32_t c = slice_cnt[i];
    if (c < 0 || c > top_k) TH_FAIL("th_merge_slices: a list count outside [0, top_k]");
    for (int32_t j = 0; j < c; ++j)
      if (!key_ok(slice_keys[i * top_k + j], doc_base)) TH_FAIL("th_merge_slices: a real key is 0 or its doc is out of range");
  }
  const size_t n_keys = (size_t)nq * n_lists * top_k, n_out = (size_t)nq * top_k;
  Bufs b;
  MergeLaunch M{};
  uint64_t* dKeys; int32_t* dCnt; uint64_t* dTheta; unsigned long long *dTotal, *dKnown; int32_t *dPruned, *dTerm;
  int32_t *dDocs, *dCounts, *dFlags; float* dScores; long long* dOutTotal;
  TH_TRY(b.upload(&dKeys, slice_keys, n_keys));
  TH_TRY(b.upload(&dCnt, slice_cnt, (size_t)nq * n_lists));
  TH_TRY(b.upload(&dTheta, theta, (size_t)nq));
  TH_TRY(b.upload(&dTotal, total_hits, (size_t)nq));
  TH_TRY(b.upload(&dKnown, known_hits, (size_t)nq));
  TH_TRY(b.upload(&dPruned, pruned, (size_t)nq));
  TH_TRY(b.upload(&dTerm, (const int32_t*)terminated, (size_t)nq));
  TH_TRY(b.upload(&dDocs, (const int32_t*)out_docs, n_out));
  TH_TRY(b.upload(&dScores, (const float*)out_scores, n_out));
  TH_TRY(b.upload(&dCounts, (const int32_t*)out_counts, (size_t)nq));
  TH_TRY(b.upload(&dOutTotal, (const long long*)out_total, (size_t)nq));
  TH_TRY(b.upload(&dFlags, (const int32_t*)out_flags, (size_t)nq));
  M.slice_keys = dKeys; M.slice_cnt = dCnt; M.n_lists = n_lists; M.top_k = top_k; M.nq = nq; M.doc_base = doc_base;
  M.out_docs = dDocs; M.out_scores = dScores; M.out_counts = dCounts;
  M.total_hits = dTotal; M.pruned = dPruned; M.terminated = dTerm; M.terminate_after = terminate_after;
  M.out_total = dOutTotal; M.out_flags = dFlags; M.known_hits = dKnown; M.theta = dTheta;
  merge_slices_kernel<<<nq, kMergeThreads>>>(M);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  TH_TRY(Bufs::download(out_docs, dDocs, n_out));
  TH_TRY(Bufs::download(out_scores, dScores, n_out));
  TH_TRY(Bufs::download(out_counts, dCounts, (size_t)nq));
  TH_TRY(Bufs::download(terminated, dTerm, (size_t)nq));
  TH_TRY(Bufs::download(out_total, dOutTotal, (size_t)nq));
  TH_TRY(Bufs::download(out_flags, dFlags, (size_t)nq));
  return 0;
}

// flush_top_k in one CTA of n_threads threads: cand[cap] (in/out) holds *count keys (a count above cap is clamped by the
// kernel), *count (in/out), *g_theta (in/out: the query's published threshold) and *theta (in/out: the CTA's copy).
TH_API int th_flush_top_k(int32_t cap, int32_t n_threads, uint64_t* cand, int32_t* count, int32_t top_k, uint64_t dec,
                          uint64_t* g_theta, uint64_t* theta) {
  if (cap <= 0 || cap > 4096 || (cap & (cap - 1)) != 0) TH_FAIL("th_flush_top_k: cap must be a power of two <= 4096");
  if (top_k <= 0 || top_k > kMaxTopK || top_k > cap) TH_FAIL("th_flush_top_k: top_k outside [1, min(cap, 1024)]");
  if (n_threads <= 0 || n_threads > 1024 || n_threads % 32 != 0) TH_FAIL("th_flush_top_k: n_threads must be a multiple of 32 <= 1024");
  if (!cand || !count || !g_theta || !theta || *count < 0) TH_FAIL("th_flush_top_k: bad argument");
  if (dec > 1) TH_FAIL("th_flush_top_k: dec must be 0 or 1");
  for (int32_t i = 0; i < *count && i < cap; ++i)
    if (!key_ok(cand[i], 0)) TH_FAIL("th_flush_top_k: a real key is 0 or its doc is negative");
  Bufs b;
  uint64_t *dCand, *dG; int32_t* dCount; unsigned long long* dTheta;
  TH_TRY(b.upload(&dCand, (const uint64_t*)cand, (size_t)cap));
  TH_TRY(b.upload(&dCount, (const int32_t*)count, 1));
  TH_TRY(b.upload(&dG, (const uint64_t*)g_theta, 1));
  TH_TRY(b.upload(&dTheta, (const unsigned long long*)theta, 1));
  flush_kernel<<<1, n_threads, (size_t)cap * sizeof(uint64_t)>>>(dCand, cap, dCount, top_k, (unsigned long long)dec, dG, dTheta);
  NRT_CUDA_TRY(cudaGetLastError());
  NRT_CUDA_TRY(cudaDeviceSynchronize());
  TH_TRY(Bufs::download(cand, dCand, (size_t)cap));
  TH_TRY(Bufs::download(count, dCount, 1));
  TH_TRY(Bufs::download(g_theta, dG, 1));
  TH_TRY(Bufs::download(theta, (const uint64_t*)dTheta, 1));
  return 0;
}
