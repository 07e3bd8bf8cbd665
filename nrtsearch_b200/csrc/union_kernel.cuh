// Union lists of multi-phrase positions (NRTGPU_MULTI_PHRASE; batch_plan.h kUnionList), built on the device for a call:
// every distinct alternative set of the batch (CompiledBatch::union_*) becomes one doc-ascending list of entries, an entry
// per doc that holds at least one alternative, with
//   - the entry's positions: the merged positions of its alternatives' postings, repeats kept (UnionPostingsEnum), for a
//     phrase position (mode 2);
//   - the entry's score: (float) of the double sum, in ascending term id order, of each present alternative's BM25 float
//     at its own weight boost * idf (a one-position MultiPhraseQuery, rewritten to SHOULD TermQuerys; mode 1).
// A fixed sequence of launches whatever the number of unions (union_build in nrtgpu.cu): gather every alternative's
// postings as (union << 32 | doc) keys, one radix sort of the keys (stable: equal docs keep their alternatives in
// ascending term id order), flag and scan the runs of equal keys (entry numbers), fill the entries (doc, score, position
// count), scan the position counts, merge each entry's positions, and write every union clause's entry range over the
// union index the host left in its post_base. Liveness is not applied here: the engine applies it when it evaluates a
// doc, as for every other list.
#pragma once
#include <cub/cub.cuh>
#include "query_eval.cuh"

namespace nrtgpu {

// what the window engine reads of the call's unions (the entries of every union, union after union)
struct UnionView {
  const int32_t* docs;       // [E] the entry's doc (the image's local doc id)
  const float* score;        // [E] mode 1: the entry's score
  const int32_t* pos_off;    // [E + 1] mode 2: entry e's positions are positions[pos_off[e], pos_off[e + 1])
  const int32_t* positions;
};

struct UnionBuildLaunch {
  DevIndexView ix;
  int32_t n_alts;
  const int64_t* alt_gstart;   // [n_alts + 1] first gathered posting of each alternative
  const int64_t* alt_post;     // [n_alts] the alternative's first posting in the image
  const int32_t* alt_term;
  const int32_t* alt_union;
  const int32_t* alt_field;    // the alternative's text field
  const float* alt_weight;     // mode 1: boost * idf
  const uint8_t* union_mode;   // [n_unions] 0: presence, 1: scored, 2: positions
  int64_t n_gather;            // S = alt_gstart[n_alts]
  const uint64_t* keys;        // [S] sorted
  const int32_t* vals;         // [S] the gathered index of each sorted key
  int32_t* head;               // [S] 1 at the first key of a run
  const int32_t* incl;         // [S] inclusive scan of head: entry number + 1
  int32_t* docs; float* score; int32_t* first;   // [S] per entry
  int32_t* npos;               // [S + 1] per entry, zeroed
  const int32_t* pos_off;      // [S + 1] exclusive scan of npos
  int32_t* positions;
  DevClause* clauses;          // the batch's clauses
  const int32_t* union_clause; int32_t n_union_clauses;
};

__device__ __forceinline__ int union_alt(const UnionBuildLaunch& U, int64_t g) {   // the alternative of gathered posting g
  int lo = 0, hi = U.n_alts;   // the last a with alt_gstart[a] <= g
  while (hi - lo > 1) { const int m = (lo + hi) >> 1; if (U.alt_gstart[m] <= g) lo = m; else hi = m; }
  return lo;
}

__global__ void union_gather_kernel(UnionBuildLaunch U, uint64_t* keys, int32_t* vals) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= U.n_gather) return;
  const int a = union_alt(U, g);
  const int32_t doc = U.ix.post_docs[U.alt_post[a] + (g - U.alt_gstart[a])];
  keys[g] = ((uint64_t)(uint32_t)U.alt_union[a] << 32) | (uint32_t)doc;
  vals[g] = (int32_t)g;
}

__global__ void union_head_kernel(UnionBuildLaunch U) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= U.n_gather) return;
  U.head[r] = (r == 0 || U.keys[r] != U.keys[r - 1]) ? 1 : 0;
}

// exact freq of image posting gp (post_f8 saturates at 255: the exception list holds the rest)
__device__ __forceinline__ float posting_freq(const DevIndexView& ix, int64_t gp) {
  const uint32_t b = ix.post_f8[gp];
  if (b < 255u) return (float)b;
  int a = 0, c = ix.n_exc;
  while (a < c) { const int m = (a + c) >> 1; if (ix.exc_pos[m] < gp) a = m + 1; else c = m; }
  return (a < ix.n_exc && ix.exc_pos[a] == gp) ? (float)ix.exc_freq[a] : 255.0f;
}

// the positions of image posting gp, alternative a's local posting lo: [*b, *e) of ix.positions
__device__ __forceinline__ void posting_positions(const UnionBuildLaunch& U, int a, int64_t lo, int64_t* b, int64_t* e) {
  const int32_t t = U.alt_term[a];
  const int64_t gp = U.alt_post[a] + lo, base = U.ix.pos_base[t];
  *b = base + U.ix.pos_off[gp];
  *e = lo + 1 < U.alt_gstart[a + 1] - U.alt_gstart[a] ? base + U.ix.pos_off[gp + 1] : U.ix.pos_base[t + 1];
}

// the entry of every run of equal keys: doc, first sorted index, score (mode 1) or position count (mode 2)
__global__ void union_entry_kernel(UnionBuildLaunch U) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= U.n_gather || !U.head[r]) return;
  const int32_t e = U.incl[r] - 1;
  const uint64_t key = U.keys[r];
  const int32_t doc = (int32_t)(uint32_t)key;
  const int mode = U.union_mode[key >> 32];
  double sum = 0.0;
  int32_t np = 0;
  for (int64_t i = r; i < U.n_gather && U.keys[i] == key; ++i) {
    const int64_t g = U.vals[i];
    const int a = union_alt(U, g);
    const int64_t lo = g - U.alt_gstart[a];
    if (mode == 1) {   // the alternative's TermQuery: BM25(boost * idf, freq, the doc's norm in its field)
      const int32_t f = U.alt_field[a];
      const uint8_t* nrm = U.ix.norms[f];
      const uint32_t nb = nrm ? (uint32_t)nrm[doc] : 1u;
      sum += (double)bm25_score(U.alt_weight[a], posting_freq(U.ix, U.alt_post[a] + lo), U.ix.caches[f * 256 + nb]);
    } else if (mode == 2) {
      int64_t b, en;
      posting_positions(U, a, lo, &b, &en);
      np += (int32_t)(en - b);
    }
  }
  U.docs[e] = doc; U.first[e] = (int32_t)r; U.npos[e] = np;
  if (mode == 1) U.score[e] = (float)sum;
}

// the merged positions of every entry of a phrase-position union: the entry's postings (one per alternative present in
// the doc) each hold an ascending run of positions, and every position is written at its rank in the merged list -- its
// index in its own run plus, per other run, the positions below it (at or below it in an earlier run, so that equal
// positions keep run order) found by binary search: O(n k log n) for n positions in k runs, no scratch
__global__ void union_positions_kernel(UnionBuildLaunch U) {
  const int64_t n_entries = U.n_gather > 0 ? U.incl[U.n_gather - 1] : 0;
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_entries) return;
  const int64_t r = U.first[e];
  const uint64_t key = U.keys[r];
  if (U.union_mode[key >> 32] != 2) return;
  int32_t* out = U.positions + U.pos_off[e];
  int64_t r_end = r;
  while (r_end < U.n_gather && U.keys[r_end] == key) ++r_end;
  auto run = [&](int64_t i, int64_t* b, int64_t* en) {   // the positions of the entry's posting i
    const int64_t g = U.vals[i];
    const int a = union_alt(U, g);
    posting_positions(U, a, g - U.alt_gstart[a], b, en);
  };
  const int32_t* P = U.ix.positions;
  for (int64_t i = r; i < r_end; ++i) {
    int64_t bi, ei;
    run(i, &bi, &ei);
    for (int64_t p = bi; p < ei; ++p) {
      const int32_t v = P[p];
      int64_t at = p - bi;
      for (int64_t j = r; j < r_end; ++j) {
        if (j == i) continue;
        int64_t lo, hi;
        run(j, &lo, &hi);
        const int64_t b0 = lo;
        while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (j < i ? P[m] <= v : P[m] < v) lo = m + 1; else hi = m; }
        at += lo - b0;
      }
      out[at] = v;
    }
  }
}

// every union clause's entry range: the entries of the keys of its union (the host left the union's index in post_base)
__global__ void union_patch_kernel(UnionBuildLaunch U) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= U.n_union_clauses) return;
  DevClause& c = U.clauses[U.union_clause[i]];
  const uint64_t u = (uint64_t)c.post_base;
  auto lower = [&](uint64_t k) {   // the first sorted key >= k
    int64_t lo = 0, hi = U.n_gather;
    while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (U.keys[m] < k) lo = m + 1; else hi = m; }
    return lo;
  };
  const int64_t r0 = lower(u << 32), r1 = lower((u + 1) << 32);
  c.post_base = r0 < r1 ? U.incl[r0] - 1 : 0;
  c.n_post = r0 < r1 ? U.incl[r1 - 1] - (U.incl[r0] - 1) : 0;
}

}  // namespace nrtgpu
