// What the host-side batch compiler / work planner (batch_plan.inc) and the kernels must agree on: the compiled clause and
// query records, the hit key, the constants that size slices, granules and term slots, and the work-item word of the
// probe kernel with the granule range and boundary entries it stands for. Standard headers only besides the C ABI, so
// that g++ compiles it as well (tests/csrc/plan_harness.cpp).
#pragma once
#include "../../include/nrtgpu.h"

#include <stdint.h>
#include <string>

#ifdef __CUDACC__
#define NRT_HD __host__ __device__ __forceinline__
#else
#include <algorithm>
#define NRT_HD inline
#endif

namespace nrtgpu {

// ---- error plumbing (thread-local message, returned through nrtgpu_last_error) ----
void set_error(const std::string& msg);
#define NRT_FAIL(code, msg) do { ::nrtgpu::set_error(msg); return (code); } while (0)

constexpr int kMaxClauses = 16;     // clauses per flat BooleanQuery on the GPU path
constexpr int kMaxTermSlots = 8;    // term clauses (tree batches: term leaves) per query: one tf byte each in the window kernel's 64-bit words
constexpr int kWindowDocs = 16384;  // window engine: W
constexpr int kSliceWindows = 64;   // window engine: windows per work item
constexpr int kWideSliceDocs = kSliceWindows * kWindowDocs;   // => 1,048,576 docs per slice of the window engine
constexpr int kMaxTopK = 1024;
constexpr int kMaxAggs = 8;         // aggregations per search
constexpr int kAggChunk = 2048;     // largest size of a terms aggregation (agg_terms_topk_kernel)
constexpr int kMaxNested = 4;       // nested collectors per terms aggregation
constexpr int kMaxNestedTopHits = 1024;               // top_hits of a nested top-hits collector (nested_top_hits_kernel)
constexpr int64_t kMaxNestedHitOutputs = 1ll << 24;   // nq * size * top_hits of one nested top-hits collector
constexpr int64_t kNestedHitBudget = 1ll << 26;       // keys (8 B) of one pass-2 group of a batch's nested top hits

struct DevClause {
  int64_t post_base;  // offset of the term's postings in post_docs / post_f8
  int32_t n_post;
  int32_t occur;
  int32_t kind;
  int32_t slot;       // byte index inside the window word (term clauses), -1 otherwise
  int32_t field;      // text field (norms + cache) for term clauses
  int32_t col;        // doc-value column for range clauses
  float weight;       // boost*idf (term) or constant score = boost (range / match-all)
  int32_t scoring;    // 1 if the clause contributes to the score (MUST / SHOULD)
  float ub;           // term clauses: largest score of any posting of the list (index-time max of tf*cache[norm])
  int32_t plane;      // term clauses: dense tf plane of the term (DevIndexView::dense_tf), -1 if the term has none
  int32_t gran_row;   // term clauses: row of the index-time granule offset table (DevIndexView::gran_tab), -1 if none
  int32_t node;       // tree batches: the child node of an NRTGPU_NODE clause, the node a leaf belongs to; 0 otherwise
                      // (col: the term id of a phrase term clause, the record of an NRTGPU_PHRASE clause)
  int64_t lo, hi;
};
static_assert(sizeof(DevClause) == 72, "DevClause layout");

// Query trees (nrtgpu_search_tree): a tree batch compiles every query into nodes in pre-order, node 0 being the root
// BooleanQuery, and lays out the clauses node after node, each node's in their given order. A node's clauses are
// cl[clause_begin, clause_begin + n_clauses) of its query (relative to DevQuery::clause_begin); child nodes follow their
// parent, so evaluating the nodes in reverse order sees every child before its parent.
constexpr int kMaxTreeClauses = 32;   // clauses of one tree, nodes and leaves
constexpr int kMaxTreeNodes = 9;      // the root and up to 8 nested nodes
constexpr int kMaxTreeDepth = 4;      // levels of queries, the root included

// CONSTANT and MIN_SCORE nodes (one MUST clause: n_req 1, need_should 0) read no msm or tie breaker, so their boost and
// threshold share those words and the record keeps its size.
struct DevNode {
  int32_t kind;           // NRTGPU_NODE_BOOL / _DISMAX / _CONSTANT / _MIN_SCORE
  int32_t clause_begin;   // relative to the query's clause_begin
  int32_t n_clauses;
  int32_t n_req;          // BOOL: MUST + FILTER clauses
  int32_t need_should;    // BOOL: minimum matching SHOULD clauses (DISMAX: 1)
  union {
    int32_t msm;          // BOOL: minimumNumberShouldMatch as given
    float min_score;      // MIN_SCORE
  };
  union {
    float tie_breaker;    // DISMAX
    float boost;          // CONSTANT / MIN_SCORE
  };
  int32_t empty;          // 1: can match nothing
};
static_assert(sizeof(DevNode) == 32, "DevNode layout");

// Phrase leaves of tree batches (nrtgpu_search_tree_phrases). Each phrase term is a presence-only term clause of its own
// slot (scoring 0, col = its term id, which indexes the image's positions), laid out after every node's clauses so that
// no node walks it; the NRTGPU_PHRASE clause holds the phrase's record index in col (relative to the query's first
// record, -1: a phrase of no terms, which matches nothing), its field and its weight. A phrase has at least two terms
// (one term is compiled as that term's leaf), so a tree of 8 term slots holds at most 4 records.
constexpr int kMaxTreePhrases = kMaxTermSlots / 2;
struct DevPhrase {
  int32_t clause0;        // its first term clause, relative to the query's clause_begin; term i is clause0 + i
  int32_t n_terms;        // 2..8, ordered by query position (stable): term 0 leads the exact matcher
  int32_t slop;
  int32_t field;
  float weight;           // boost * (float) sum of the terms' idf (double sum)
  int32_t cover_slot;     // the slot of its rarest term
  int32_t reserved[2];
  int32_t offset[kMaxTermSlots];   // PhraseQuery positions of the terms
};
static_assert(sizeof(DevPhrase) == 64, "DevPhrase layout");

// Multi-phrase leaves of tree batches (NRTGPU_MULTI_PHRASE, nrtgpu_search_tree_phrases). A position that holds several
// alternative terms takes ONE term slot whose list is a union built on the device for the call (union_kernel.cuh): a
// term clause (kind NRTGPU_TERM) with plane kUnionList, post_base / n_post its range of the call's union entries (the
// host writes the union's index into post_base, union_patch_kernel the range). A one-position multi-phrase is such a
// slot on its own, scored from the union's per-entry score (SHOULD TermQuerys over the alternatives); a longer one is a
// DevPhrase whose union positions read the union's merged positions. Only the kUnion instantiations of the window
// engine read plane there; every other engine refuses the kind.
constexpr int32_t kUnionList = -2;
constexpr int kMaxUnionAlternatives = 128;        // alternatives of one multi-phrase position
constexpr int64_t kMaxUnionPostings = 1ll << 25;  // postings the distinct unions of one call gather (52 B each of scratch)
constexpr int64_t kMaxUnionPositions = 1ll << 27; // positions the distinct phrase-position unions of one call merge (4 B each)

// Block joins of tree batches (NRTGPU_NODE_NESTED). compile_tree compiles each join's child query as an extra query of the
// batch, after the request's nq (query nq + j is join j's), and the clause that referenced the join as a term slot of
// plane kUnionList whose list is the join's (parent, score) entries, built on the device behind the union entries
// (join_kernel.cuh; the host writes the join's index into post_base, join_patch_kernel the range). Each join's child
// matches are bounded by the postings of its child query's driver lists, and the bounds of one call by kMaxJoinChildren.
constexpr int64_t kMaxJoinChildren = 1ll << 26;   // bounded child matches of one call (40 B each of scratch)

struct DevQuery {
  int32_t clause_begin, n_clauses;
  int32_t n_term;          // number of term clauses (= slots used)
  int32_t n_req;           // MUST + FILTER clauses (all kinds)
  int32_t need_should;     // minimum matching SHOULD clauses
  int32_t msm;             // minimumNumberShouldMatch as given
  uint32_t req_term_mask;  // bit s set: term slot s is MUST/FILTER
  uint32_t not_term_mask;  // bit s set: term slot s is MUST_NOT
  uint32_t driver_mask;    // bit s set: term slot s drives pass 2
  int32_t dense_driver;    // 1: iterate every doc of the window instead of driver postings
  int32_t has_non_driver;  // 1: some term slot is not a driver (pass 3 needed)
  int32_t has_nonterm;     // 1: range / match-all clauses present
  int32_t empty;           // 1: can match nothing
  int32_t has_after;
  uint32_t must_term_mask;    // bit s set: term slot s is MUST (scores into the required sum)
  uint32_t should_term_mask;  // bit s set: term slot s is SHOULD
  int32_t nonterm_scoring;    // 1: a range / match-all clause is MUST or SHOULD (contributes a constant score)
  int32_t single_field;       // >= 0: every term clause reads this text field's norms; -1: mixed
  uint64_t after_key;
};
static_assert(sizeof(DevQuery) == 80, "DevQuery layout");

// ---- total order on hits: (score desc, doc asc)  <=>  key desc ----
// reference: src/main/java/org/apache/lucene/search/LazyQueueTopScoreDocCollector.java:129-143
// key = ordered(score) << 32 | ~doc ; all keys of real hits are > 0, so 0 is the "empty" sentinel.
NRT_HD uint32_t float_to_ordered(float f) {
#ifdef __CUDA_ARCH__
  uint32_t b = __float_as_uint(f);
#else
  union { float f; uint32_t u; } c; c.f = f; uint32_t b = c.u;
#endif
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
NRT_HD float ordered_to_float(uint32_t u) {
  uint32_t b = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  union { float f; uint32_t u; } c; c.u = b; return c.f;
#endif
}
NRT_HD uint64_t make_key(float score, int32_t doc) {
  return ((uint64_t)float_to_ordered(score) << 32) | (uint32_t)(~(uint32_t)doc);
}
NRT_HD float key_score(uint64_t k) { return ordered_to_float((uint32_t)(k >> 32)); }
NRT_HD int32_t key_doc(uint64_t k) { return (int32_t)(~(uint32_t)k); }

namespace v3 {
#ifndef __CUDACC__
using std::max;
using std::min;
#endif

constexpr int kT = 4;                       // term slots of the probe kernel (queries of up to 4 term clauses)
constexpr int kCtasA = 3;                    // resident CTAs per SM of the probe kernel's configuration A (probe_kernel.cuh)
constexpr int kLogGran = 10;                 // 1024-doc granules: the granularity of the index-time skip data (gran_tab)
constexpr int kGran = 1 << kLogGran;
constexpr int kMaxSliceGran = 512;           // a slice spans at most 512K docs (its granule offsets live in shared memory)
constexpr int kWarmGran = 32;                // granules (32K docs) of the warm-up work item of a query
constexpr int kProbeMaxTopK = 512;           // largest top_k of the probe kernel (half its candidate buffer)

// ---- per-query record of the probe kernel ----
// Everything a work item's set-up needs that depends on (query, index image) only, built on the device once per prepared
// batch (probe_query_kernel) and copied into shared memory by every item of the query; the item adds its posting bounds,
// its granule offsets and the roles that follow from the query's threshold. The record points into the index image and
// holds floats derived from its length caches: it is valid for the statistics the batch was prepared with, like the
// compiled weight / ub of its clauses.
struct alignas(16) DevProbeQuery {
  // per term slot (a slot without a term clause: kind kAbsent, NULL pointers, row -1)
  const int32_t* gdocs[kT];        // global postings of the list
  const uint8_t* gf8[kT];
  const uint8_t* plane[kT];        // byte plane (exact min(tf, 255) per doc) of the list, or NULL
  const uint8_t* plane2[kT];       // 2-bit plane (min(tf, 3), four docs per byte): what the probes gather
  float weight[kT];
  float ub[kT];
  int32_t kind[kT];                // kPlane / kLong / kShort / kAbsent (an item may turn kShort into kGlobal)
  int32_t clause[kT];
  int32_t field[kT];
  uint32_t pbm[kT];                // post_base mod 16 (alignment of the list inside the global posting arrays)
  int32_t row[kT];                 // row of the index-time granule offsets, -1: none
  // MAXSCORE order: the slots ascending by ub (equal bounds in slot order) and the float of the running double sum of
  // their bounds; the non-essential lists of an item are the longest prefix with pre[a] < theta.score
  int32_t ord[kT];
  float pre[kT];
  DevQuery q;
  DevClause cl[kMaxClauses];
  float ubt[256];                  // pure disjunctions: score bound per tf pattern, index sum min(tf_s, 3) * 4^s
  // pure disjunctions, exact sweep warm-up (TOP_SCORES, every other slot has a plane): the warm-up scores the docs of
  // warm_slot's list below granule warm_gran exactly and outputs them; the query's other items leave those postings to
  // it. warm_slot -1 and warm_gran 0: none.
  int32_t warm_slot;
  int32_t warm_gran;
  int32_t reserved[2];
};
static_assert(sizeof(DevProbeQuery) % 16 == 0, "DevProbeQuery is copied 16 bytes at a time");

// ---- work item of the probe kernel: slice | part << 16 | log2(parts) << 20 | flags << 24 ----
// A (query, slice) is split into 2^lparts parts of equal granule ranges; part p covers the finest parts
// [p * kfine, (p + 1) * kfine) of the slice's parts_max, kfine = parts_max >> lparts.
enum : int {
  kItemWarmDocs = 1,     // warm-up item: the first kWarmGran granules of slice 0
  kItemBehindWarm = 2,   // slice-0 item of a query with a warm-up item: starts behind those granules
  kItemSweep = 4,        // sweep warm-up item: the first 32K postings of one list over the whole shard (slot in the part bits)
};
NRT_HD int32_t item_encode(int slice, int part, int lparts, int flags) {
  return slice | (part << 16) | (lparts << 20) | (flags << 24);
}
NRT_HD int32_t item_encode_sweep(int slot) { return item_encode(0, slot, 0, kItemSweep); }
NRT_HD int item_slice(int32_t w) { return w & 0xffff; }
NRT_HD int item_flags(int32_t w) { return w >> 24; }
NRT_HD int item_sweep_slot(int32_t w) { return (w >> 16) & 0xf; }
NRT_HD int item_part(int32_t w) { return (item_flags(w) & kItemSweep) ? 0 : ((w >> 16) & 0xf); }
NRT_HD int item_lparts(int32_t w) { return (w >> 20) & 0xf; }

// Boundary entries per (query, term slot) (sbounds of slice_bounds_kernel): n_slices * parts_max part boundaries
// (slice-major), the shard end, the end of the warm-up granules of slice 0, the end of the exact sweep warm-up
// (DevProbeQuery::warm_gran, a per-query granule).
NRT_HD int boundary_end_entry(int n_slices, int parts_max) { return n_slices * parts_max; }
NRT_HD int boundary_warm_entry(int n_slices, int parts_max) { return n_slices * parts_max + 1; }
NRT_HD int boundary_exact_entry(int n_slices, int parts_max) { return n_slices * parts_max + 2; }
NRT_HD int boundary_entries(int n_slices, int parts_max) { return n_slices * parts_max + 3; }
constexpr uint32_t kSweepPostings = 32768;   // postings of the rarest list a sweep warm-up scores (at least, when exact)

// Granules [g_lo, g_hi) of the item inside its slice (g_count granules, parts_max finest parts of `fine` granules each),
// and the boundary entries e_lo / e_hi that hold its lists' posting bounds. A kItemBehindWarm item also starts at or after
// the warm-up entry's postings. A sweep item has whole-shard bounds (entry 0 to the shard end) and one dummy granule.
struct ItemSpan { int g_lo, g_hi, e_lo, e_hi; };
NRT_HD ItemSpan item_span(int32_t w, int g_count, int fine, int parts_max, int n_slices) {
  const int slice = item_slice(w), flags = item_flags(w), part = item_part(w);
  const int kfine = parts_max >> item_lparts(w);   // finest parts per part of this item
  ItemSpan r;
  r.g_lo = min(g_count, part * kfine * fine);
  r.g_hi = ((part + 1) * kfine >= parts_max) ? g_count : min(g_count, (part + 1) * kfine * fine);
  r.e_lo = slice * parts_max + part * kfine;
  r.e_hi = slice * parts_max + (part + 1) * kfine;   // (part + 1) * kfine == parts_max: entry 0 of the next slice / the end entry
  if (flags & kItemBehindWarm) r.g_lo = max(r.g_lo, min(g_count, kWarmGran));
  if (flags & kItemWarmDocs) { r.g_hi = min(g_count, kWarmGran); r.e_hi = boundary_warm_entry(n_slices, parts_max); }
  if (flags & kItemSweep) { r.g_lo = 0; r.g_hi = 1; r.e_lo = 0; r.e_hi = boundary_end_entry(n_slices, parts_max); }
  return r;
}
// candidate list an item writes: its first finest part's list, or the last list (warm-up items)
NRT_HD int item_out_list(int32_t w, int parts_max, int n_lists) {
  return (item_flags(w) & (kItemWarmDocs | kItemSweep)) ? n_lists - 1
                                                        : item_slice(w) * parts_max + item_part(w) * (parts_max >> item_lparts(w));
}
// shard-wide granule of boundary entry e
NRT_HD int64_t boundary_gran(int e, int n_slices, int parts_max, int slice_gran, int n_gran) {
  const int n_b = n_slices * parts_max;
  const int fine = (slice_gran + parts_max - 1) / parts_max;
  int64_t gran;
  if (e < n_b) gran = (int64_t)(e / parts_max) * slice_gran + min(slice_gran, (e % parts_max) * fine);
  else if (e == n_b) gran = n_gran;
  else gran = min(kWarmGran, slice_gran);
  if (gran > n_gran) gran = n_gran;
  return gran;
}

}  // namespace v3
}  // namespace nrtgpu
