// Block joins of tree batches (NRTGPU_NODE_NESTED; batch_plan.h kMaxJoinChildren): every join of the batch becomes one
// doc-ascending list of (parent, score) entries, written behind the call's union entries (union_kernel.cuh UnionView), so
// that the parent query reads it as a union term slot. The child pass (bool_window_emit_kernel, bool_kernel.cuh) appends
// every match of every join's child query as a (join << 32 | child doc) key and its float score; the keys beyond the
// matches hold the sentinel ~0. Then a fixed sequence of launches whatever the number of joins (join_build in nrtgpu.cu):
// one radix sort of the keys, the run heads where (join, parent) changes, the library's int scan of the heads (entry
// numbers), one thread per entry folding its run in child doc order, and every join clause's entry range over the join
// index the host left in its post_base. Liveness is not applied here: the child pass reads no live docs (Lucene's child
// scorer does not read acceptDocs), and the parent pass applies the parent's as for every other hit.
#pragma once
#include <cub/cub.cuh>
#include "query_eval.cuh"

namespace nrtgpu {

// the parent bitset of an image (nrtgpu_index_add_parents): bit d set iff doc d holds the root term
__global__ void parent_bits_kernel(const int32_t* docs, int64_t n, uint32_t* bits) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t d = docs[i];
  atomicOr(bits + (d >> 5), 1u << (d & 31));
}

struct JoinBuildLaunch {
  const uint32_t* parent_bits;   // the image's parents
  int32_t n_words;               // words of parent_bits: (n_docs + 31) / 32
  int32_t n_joins;
  int64_t n;                     // keys sorted: the matches, then the sentinels
  const uint64_t* keys;
  const float* scores;
  int32_t* head;                 // [n] 1 at the first child of a (join, parent) run
  const int32_t* incl;           // [n] inclusive scan of head: entry number + 1
  const uint8_t* mode;           // [n_joins] NRTGPU_NESTED_*
  int64_t base;                  // the first entry of the joins in the entry arrays (behind the union entries)
  int32_t* docs; float* score;   // the entry arrays (UnionView)
  DevClause* clauses;            // the batch's clauses
  const int32_t* join_clause;
};

// ToParentBlockJoinQuery's parentBits.nextSetBit(child + 1): the smallest parent doc > c, -1 when c is itself a parent
// (Lucene throws there; the reference never reaches it) or no parent follows it
__device__ __forceinline__ int32_t join_parent_of(const JoinBuildLaunch& J, uint32_t c) {
  int w = (int)(c >> 5);
  if ((__ldg(J.parent_bits + w) >> (c & 31)) & 1u) return -1;
  uint32_t m = __ldg(J.parent_bits + w) & ((c & 31) == 31 ? 0u : ~0u << ((c & 31) + 1));
  while (m == 0) {
    if (++w >= J.n_words) return -1;
    m = __ldg(J.parent_bits + w);
  }
  return w * 32 + __ffs(m) - 1;
}

// a key's join (the sentinel's is >= n_joins) and child doc
__device__ __forceinline__ uint32_t join_of(uint64_t k) { return (uint32_t)(k >> 32); }

__global__ void join_head_kernel(JoinBuildLaunch J) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= J.n) return;
  const uint64_t k = J.keys[r];
  int h = 0;
  if (join_of(k) < (uint32_t)J.n_joins) {
    const int32_t p = join_parent_of(J, (uint32_t)k);
    if (p >= 0) {
      h = 1;
      if (r > 0) {
        const uint64_t k0 = J.keys[r - 1];
        h = join_of(k0) != join_of(k) || join_parent_of(J, (uint32_t)k0) != p;
      }
    }
  }
  J.head[r] = h;
}

// the entry of every run: its parent, and the fold of its children's float scores in child doc order (BlockJoinScorer)
__global__ void join_entry_kernel(JoinBuildLaunch J) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= J.n || !J.head[r]) return;
  const int64_t e = J.base + J.incl[r] - 1;
  const uint64_t k = J.keys[r];
  const uint32_t j = join_of(k);
  const int32_t p = join_parent_of(J, (uint32_t)k);
  const int mode = J.mode[j];
  double sum = 0.0;
  float mx = J.scores[r], mn = J.scores[r];
  int64_t n = 0;
  // the run: the keys of join j whose child lies below p (no parent lies between the run's first child and p)
  for (int64_t i = r; i < J.n && join_of(J.keys[i]) == j && (int32_t)(uint32_t)J.keys[i] < p; ++i) {
    const float s = J.scores[i];
    sum += (double)s;
    mx = fmaxf(mx, s); mn = fminf(mn, s);
    ++n;
  }
  float out = 0.0f;
  if (mode == NRTGPU_NESTED_SUM) out = (float)sum;
  else if (mode == NRTGPU_NESTED_AVG) out = (float)(sum / (double)n);
  else if (mode == NRTGPU_NESTED_MAX) out = mx;
  else if (mode == NRTGPU_NESTED_MIN) out = mn;
  J.docs[e] = p;
  J.score[e] = out;
}

// every join clause's entry range: the entries of the keys of its join (the host left the join's index in post_base)
__global__ void join_patch_kernel(JoinBuildLaunch J) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= J.n_joins) return;
  DevClause& c = J.clauses[J.join_clause[i]];
  const uint64_t j = (uint64_t)c.post_base;
  auto lower = [&](uint64_t k) {   // the first sorted key >= k
    int64_t lo = 0, hi = J.n;
    while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (J.keys[m] < k) lo = m + 1; else hi = m; }
    return lo;
  };
  const int64_t r0 = lower(j << 32), r1 = lower((j + 1) << 32);
  const int64_t e0 = r0 > 0 ? J.incl[r0 - 1] : 0, e1 = r1 > 0 ? J.incl[r1 - 1] : 0;
  c.post_base = J.base + e0;
  c.n_post = (int32_t)(e1 - e0);
}

}  // namespace nrtgpu
