// One query on one doc: the device view of the index that every query kernel reads, the doc-value range test, the exact
// tf of a saturated posting, the flat clause rule shared by the window engine (bool_kernel.cuh), the generic probe kernel
// (probe_kernel.cuh) and the second pass (collect_kernel.cuh), and the query-tree walk with its phrase matcher shared by
// the window engine's tree instantiation and the second pass of tree batches. The engines differ only in how they find a
// term's tf and norm, and a phrase term's posting; each passes that in.
#pragma once
#include <type_traits>
#include "common.cuh"
#include "../../include/nrtgpu.h"

namespace nrtgpu {

// Whether a tree engine's shared state (Smem) may hold term slots whose lists are call unions (batch_plan.h kUnionList):
// only the kUnion instantiations of the window engine (bool_kernel.cuh BoolTreeSmemU), which specialise it. Every other
// engine compiles the code below without the union branches.
template <class Smem> struct SmemUnions : std::false_type {};

struct DevIndexView {
  int32_t n_docs;
  int32_t doc_base;
  const int32_t* post_docs;
  const uint8_t* post_f8;        // min(freq, 255)
  const int64_t* exc_pos;        // sorted global posting indices with freq >= 255
  const int32_t* exc_freq;
  int32_t n_exc;
  const uint8_t* const* norms;   // [n_fields] device pointers (NULL = omitNorms)
  const float* caches;           // [n_fields][256]
  const int64_t* const* col64;   // [n_columns] (NULL if stored as int32)
  const int32_t* const* col32;   // [n_columns] (NULL if stored as int64)
  const uint8_t* const* col_has; // [n_columns] (NULL = all)
  const int64_t* const* colmv_off;  // [n_columns] multi-valued columns (SORTED_NUMERIC): doc d holds colmv_val[c][off[d] .. off[d + 1]),
  const int64_t* const* colmv_val;  //              ascending; NULL entry = single-valued column
  const uint32_t* live_bits;     // bitmap or NULL
  const uint32_t* gran_tab;      // [n_rows][n_gran + 1] postings of the term below each 1024-doc granule boundary (skip data)
  int32_t n_gran;
  const uint8_t* dense_tf;       // [n_planes][dense_stride] min(freq, 255) per doc for the densest terms (0 = absent)
  int64_t dense_stride;
  const uint8_t* dense_tf2;      // [n_planes][dense_stride / 4] min(freq, 3) in 2 bits per doc: the planes the probe kernel gathers
                                 // (a quarter of the L2 / DRAM footprint of the byte planes; 3 = "three or more")
  // term positions (nrtgpu_index_add_positions; NULL without): posting p of term t holds positions[pos_base[t] + pos_off[p]
  // .. end), end = the next posting's start, or pos_base[t + 1] for the term's last posting (its exact freq positions)
  const int32_t* positions;
  const uint32_t* pos_off;       // [P]
  const int64_t* pos_base;       // [n_terms + 1]
  // keyword columns (nrtgpu_index_add_keyword_columns; NULL without): codes 2i + 2 of ordinal i, 0 = no value, per doc
  // (SORTED: kw_off[k] NULL) or per value behind the doc offsets kw_off[k] (SORTED_SET, ascending within a doc)
  const uint32_t* const* kw_codes;
  const int64_t* const* kw_off;
};

// numeric range clause on one doc (IndexOrDocValuesQuery's doc-values side, reference IntFieldDef.java:124-158 inclusive
// bounds): single-valued column = the value is in [lo, hi]; multi-valued (SortedNumericDocValuesRangeQuery) = ANY value is
__device__ __forceinline__ bool range_matches(const DevIndexView& ix, int col, int32_t doc, int64_t lo, int64_t hi) {
  const int64_t* off = ix.colmv_off ? ix.colmv_off[col] : nullptr;
  if (off) {
    const int64_t* v = ix.colmv_val[col];
    int64_t a = off[doc], b = off[doc + 1];
    while (a < b) { const int64_t m = (a + b) >> 1; if (v[m] < lo) a = m + 1; else b = m; }   // values of a doc are sorted
    return a < off[doc + 1] && v[a] <= hi;
  }
  const uint8_t* has = ix.col_has[col];
  if (has && !has[doc]) return false;
  const int64_t x = ix.col32[col] ? (int64_t)__ldg(ix.col32[col] + doc) : __ldg(ix.col64[col] + doc);
  return x >= lo && x <= hi;
}

// keyword range clause on one doc (NRTGPU_KEYWORD_RANGE: TermRangeQuery / PrefixQuery over ordinals in byte order, lo >= 1
// as compiled, so a doc without a value -- code 0 -- never matches): SORTED = its code is in [lo, hi]; SORTED_SET = ANY of
// its codes is, found as range_matches finds a multi-valued value
__device__ __forceinline__ bool keyword_codes_match(const uint32_t* v, const int64_t* off, int32_t doc, int64_t lo, int64_t hi) {
  if (off) {
    int64_t a = off[doc], b = off[doc + 1];
    const int64_t end = b;
    while (a < b) { const int64_t m = (a + b) >> 1; if ((int64_t)__ldg(v + m) < lo) a = m + 1; else b = m; }
    return a < end && (int64_t)__ldg(v + a) <= hi;
  }
  const int64_t x = (int64_t)__ldg(v + doc);
  return x >= lo && x <= hi;
}
__device__ __forceinline__ bool keyword_matches(const DevIndexView& ix, int col, int32_t doc, int64_t lo, int64_t hi) {
  return keyword_codes_match(ix.kw_codes[col], ix.kw_off[col], doc, lo, hi);
}

// keyword_matches out of line: the flat clause rule's hot loop then keeps the numeric range test as it was, and only a
// keyword clause pays the call
__device__ __noinline__ bool keyword_matches_call(const DevIndexView& ix, const DevClause& c, int32_t doc) {
  return keyword_matches(ix, c.col, doc, c.lo, c.hi);
}

// a doc-value clause (numeric or keyword range) on one doc
__device__ __forceinline__ bool dv_clause_matches(const DevIndexView& ix, const DevClause& c, int32_t doc) {
  return c.kind == NRTGPU_RANGE_I64 ? range_matches(ix, c.col, doc, c.lo, c.hi) : keyword_matches(ix, c.col, doc, c.lo, c.hi);
}
__device__ __forceinline__ bool is_dv_clause(int kind) { return kind == NRTGPU_RANGE_I64 || kind == NRTGPU_KEYWORD_RANGE; }

// exact tf of posting (clause c, doc) when the byte saturated: find the posting, then the exception list
__device__ __noinline__ float exact_freq_slow(const DevIndexView& ix, const DevClause& c, int32_t doc) {
  const int32_t* docs = ix.post_docs + c.post_base;
  int lo = 0, hi = c.n_post;
  while (lo < hi) { int m = (lo + hi) >> 1; if (docs[m] < doc) lo = m + 1; else hi = m; }
  int64_t gp = c.post_base + lo;
  int a = 0, b = ix.n_exc;
  while (a < b) { int m = (a + b) >> 1; if (ix.exc_pos[m] < gp) a = m + 1; else b = m; }
  if (a < ix.n_exc && ix.exc_pos[a] == gp) return (float)ix.exc_freq[a];
  return 255.0f;
}

// Matches and scores doc against the n_clauses clauses cl of q with Lucene's BooleanScorerSupplier rule: an absent MUST /
// FILTER clause or a present MUST_NOT clause rejects the doc, at least need_should SHOULD clauses must match, each clause
// scores a float, the MUST and SHOULD sums are doubles added in clause order, and required + optional is
// ReqOptSumScorer's float add (msm == 0) or ConjunctionScorer's double add (msm > 0).
//   term_mask: bit s set iff term slot s is present, for an engine that knows it before scoring (a doc missing a required
//              slot or holding an excluded one is rejected at once); an engine that does not passes q.req_term_mask.
//   term(c, &s): whether term clause c is present in doc; if it is and c.scoring, sets s to its BM25 float.
// Doc-value clauses (numeric and keyword ranges) and match-all clauses are evaluated before any term is scored: a doc that
// fails a required range (or holds an excluded one) costs no norm gather, as ConjunctionDISI advances the cheapest
// iterators first. They have no side effects and the sums stay in clause order, so the order changes no result.
template <class TermScore>
__device__ __forceinline__ bool eval_clauses(const DevIndexView& ix, const DevQuery& q, const DevClause* cl,
                                             int32_t doc, uint32_t term_mask, TermScore term, float* out_score) {
  if ((term_mask & q.req_term_mask) != q.req_term_mask) return false;
  if (term_mask & q.not_term_mask) return false;
  if (ix.live_bits && !((ix.live_bits[doc >> 5] >> (doc & 31)) & 1u)) return false;
  uint32_t nonterm_present = 0;   // bit i: clause i is a doc-value clause that matches, or a match-all clause
  if (q.has_nonterm)
    for (int i = 0; i < q.n_clauses; ++i) {
      const DevClause& c = cl[i];
      if (c.kind == NRTGPU_TERM) continue;
      const bool p = c.kind == NRTGPU_RANGE_I64 ? range_matches(ix, c.col, doc, c.lo, c.hi)
                   : c.kind == NRTGPU_KEYWORD_RANGE ? keyword_matches_call(ix, c, doc) : true;
      if (p) { if (c.occur == NRTGPU_MUST_NOT) return false; nonterm_present |= 1u << i; }
      else if (c.occur == NRTGPU_MUST || c.occur == NRTGPU_FILTER) return false;
    }
  double must_sum = 0.0, should_sum = 0.0;
  int n_should = 0;
  for (int i = 0; i < q.n_clauses; ++i) {
    const DevClause& c = cl[i];
    bool present;
    float s = 0.0f;
    if (c.kind == NRTGPU_TERM) {
      present = term(c, &s);
    } else {
      present = (nonterm_present >> i) & 1u;
      s = c.weight;
    }
    if (!present) {
      if (c.occur == NRTGPU_MUST || c.occur == NRTGPU_FILTER) return false;
      continue;
    }
    switch (c.occur) {
      case NRTGPU_MUST: must_sum += (double)s; break;
      case NRTGPU_FILTER: break;
      case NRTGPU_SHOULD: should_sum += (double)s; ++n_should; break;
      default: return false;   // MUST_NOT present
    }
  }
  if (n_should < q.need_should) return false;
  float score;
  if (q.n_req == 0) score = (float)should_sum;
  else {
    const float req = (float)must_sum;
    if (n_should == 0) score = req;
    else {
      const float opt = (float)should_sum;
      score = (q.msm > 0) ? (float)((double)req + (double)opt) : __fadd_rn(req, opt);
    }
  }
  *out_score = score;
  return true;
}

// One node of a query tree (tree batches: the window engine, the second pass) on one doc, its child nodes already evaluated: node_match
// bit n is set iff node n matched, node_score[n] is then the float its Scorer returned. The clauses are walked in order.
//   BOOL:   eval_clauses's rule, a child node counting as a clause that is present when it matched and scores its float;
//   DISMAX: matches if any disjunct does; DisjunctionMaxScorer's float max and double sum of the others, streamed in clause
//           order as Lucene 10 streams its disjuncts (a new max moves the old one into the sum), scored
//           (float)((double)max + others * (double)tie_breaker);
//   CONSTANT: its one MUST clause matches; scores the node's boost (the clause was compiled non-scoring);
//   MIN_SCORE: its one MUST clause matches with a float s >= min_score (MinThresholdQuery / MinScoreWrapper); scores
//           s * boost in float.
// term(c, &s) as for eval_clauses, for term and phrase leaves alike. Liveness is the caller's.
template <class TermScore>
__device__ __forceinline__ bool eval_node(const DevIndexView& ix, const DevNode& nd, const DevClause* cl, int32_t doc,
                                          uint32_t node_match, const float* node_score, TermScore term, float* out_score) {
  double must_sum = 0.0, should_sum = 0.0;
  float max_s = 0.0f;
  int n_should = 0;
  for (int i = 0; i < nd.n_clauses; ++i) {
    const DevClause& c = cl[nd.clause_begin + i];
    bool present;
    float s = 0.0f;
    if (c.kind == NRTGPU_TERM || c.kind == NRTGPU_PHRASE) {
      present = term(c, &s);
    } else if (is_dv_clause(c.kind)) {
      present = dv_clause_matches(ix, c, doc);
      s = c.weight;
    } else if (c.kind == NRTGPU_NODE) {
      present = (node_match >> c.node) & 1u;
      if (present) s = node_score[c.node];
    } else {
      present = true;
      s = c.weight;
    }
    if (!present) {
      if (c.occur == NRTGPU_MUST || c.occur == NRTGPU_FILTER) return false;
      continue;
    }
    switch (c.occur) {
      case NRTGPU_MUST: must_sum += (double)s; break;
      case NRTGPU_FILTER: break;
      case NRTGPU_SHOULD:
        if (nd.kind == NRTGPU_NODE_DISMAX) {
          if (s >= max_s) { should_sum += (double)max_s; max_s = s; }
          else should_sum += (double)s;
        } else should_sum += (double)s;
        ++n_should;
        break;
      default: return false;   // MUST_NOT present
    }
  }
  if (n_should < nd.need_should) return false;
  float score;
  if (nd.kind == NRTGPU_NODE_DISMAX) score = (float)((double)max_s + should_sum * (double)nd.tie_breaker);
  else if (nd.kind == NRTGPU_NODE_CONSTANT) score = nd.boost;
  else if (nd.kind == NRTGPU_NODE_MIN_SCORE) {
    const float s = (float)must_sum;   // its one MUST clause's float
    if (!(s >= nd.min_score)) return false;   // hasPassedMinScore: s > min || s == min (NaN: never)
    score = __fmul_rn(s, nd.boost);
  }
  else if (nd.n_req == 0) score = (float)should_sum;
  else {
    const float req = (float)must_sum;
    if (n_should == 0) score = req;
    else {
      const float opt = (float)should_sum;
      score = (nd.msm > 0) ? (float)((double)req + (double)opt) : __fadd_rn(req, opt);
    }
  }
  *out_score = score;
  return true;
}

// bit s set: byte s (term slot s) of a slot word is non-zero
__device__ __forceinline__ uint32_t presence_mask(uint64_t s) {
  uint32_t m = 0;
#pragma unroll
  for (int i = 0; i < kMaxTermSlots; ++i) m |= (((s >> (8 * i)) & 0xff) != 0 ? 1u : 0u) << i;
  return m;
}

// The freq of phrase ph in doc, which holds every term of it (PhraseScorer: the sum of sloppyWeight over the matches), or
// with first_only 1 as soon as one match is found (a phrase under FILTER / MUST_NOT only has to match); 0: no match.
// Term i's posting is phrase_posting(ix, sm, term clause, doc), the engine's (its index in the term's list); its positions are
// the posting's range of the image's positions. Fixed-size per-thread state, no recursion.
//   slop 0: ExactPhraseMatcher: every position of the lead (term 0, the smallest query position) at which each other term
//           has the position lead - offset[0] + offset[j] counts 1;
//   slop>0: SloppyPhraseMatcher without repeats: the PhraseQueue of (position - offset, offset, ordinal) -- a total order, so
//           a scan for its minimum pops what the heap pops --, the running end and the match-length minimisation; every
//           match adds 1.0f / (1.0f + matchLength) in float.
template <class Smem>
__device__ __noinline__ float phrase_freq(const DevIndexView& ix, const Smem& sm, const DevPhrase& ph, int32_t doc,
                                          bool first_only) {
  constexpr bool kUnions = SmemUnions<Smem>::value;
  const int n = ph.n_terms;
  int64_t cur[kMaxTermSlots], end[kMaxTermSlots];
  const int32_t* P = ix.positions;
  uint32_t in_union = 0;   // (kUnions) bit i: term i's positions are sm.u.positions[cur[i] .. end[i]), else P's
  auto at = [&](int i, int64_t k) {   // position k of term i
    if constexpr (kUnions) return __ldg(((in_union >> i) & 1u ? sm.u.positions : P) + k);
    else return __ldg(P + k);
  };
  for (int i = 0; i < n; ++i) {
    const DevClause& t = sm.cl[ph.clause0 + i];
    const uint32_t lo = phrase_posting(ix, sm, t, doc);
    if constexpr (kUnions) {
      if (t.plane == kUnionList) {   // a union slot: its entry's merged positions
        const int64_t e = t.post_base + lo;
        in_union |= 1u << i;
        cur[i] = __ldg(sm.u.pos_off + e);
        end[i] = __ldg(sm.u.pos_off + e + 1);
        continue;
      }
    }
    const int64_t gp = t.post_base + lo, base = __ldg(ix.pos_base + t.col);
    cur[i] = base + __ldg(ix.pos_off + gp);
    end[i] = (int64_t)lo + 1 < (int64_t)t.n_post ? base + __ldg(ix.pos_off + gp + 1) : __ldg(ix.pos_base + t.col + 1);
  }
  float freq = 0.0f;
  if (ph.slop == 0) {
    for (int64_t a = cur[0]; a < end[0]; ++a) {
      const int32_t phrase_pos = at(0, a) - ph.offset[0];
      bool ok = true;
      for (int j = 1; j < n && ok; ++j) {
        const int32_t want = phrase_pos + ph.offset[j];
        while (cur[j] < end[j] && at(j, cur[j]) < want) ++cur[j];
        if (cur[j] == end[j]) return freq;   // term j has no position left: no later lead position can match
        ok = at(j, cur[j]) == want;
      }
      if (ok) { freq = __fadd_rn(freq, 1.0f); if (first_only) return freq; }
    }
    return freq;
  }
  int32_t pos[kMaxTermSlots];
  int32_t end_pos = INT_MIN;
  uint32_t inq = 0;
  for (int i = 0; i < n; ++i) {
    pos[i] = at(i, cur[i]) - ph.offset[i]; ++cur[i];
    end_pos = max(end_pos, pos[i]);
    inq |= 1u << i;
  }
  auto top = [&](uint32_t m) {   // the queue's least element: position, then offset, then ordinal
    int best = -1;
    for (int i = 0; i < n; ++i) {
      if (!((m >> i) & 1u)) continue;
      if (best < 0 || pos[i] < pos[best] || (pos[i] == pos[best] && ph.offset[i] < ph.offset[best])) best = i;
    }
    return best;
  };
  for (;;) {   // nextMatch
    int pp = top(inq);
    inq &= ~(1u << pp);
    int32_t match_len = end_pos - pos[pp];
    int32_t next = pos[top(inq)];
    bool positioned = true, matched = false;
    for (;;) {
      if (cur[pp] >= end[pp]) { positioned = false; matched = match_len <= ph.slop; break; }
      pos[pp] = at(pp, cur[pp]) - ph.offset[pp]; ++cur[pp];
      end_pos = max(end_pos, pos[pp]);
      if (pos[pp] > next) {   // done minimising the current match length
        inq |= 1u << pp;
        if (match_len <= ph.slop) { matched = true; break; }
        pp = top(inq);
        inq &= ~(1u << pp);
        next = pos[top(inq)];
        match_len = end_pos - pos[pp];
      } else {
        match_len = min(match_len, end_pos - pos[pp]);
      }
    }
    if (!matched) return freq;
    freq = __fadd_rn(freq, __fdiv_rn(1.0f, __fadd_rn(1.0f, (float)match_len)));
    if (first_only || !positioned) return freq;
  }
}

// The query tree staged in sm on one doc whose slot word holds the tf byte of every term slot (0: absent; phrase terms and
// terms that do not score: 1): the root's required and excluded slots, liveness, then the nodes bottom-up (reverse
// pre-order: children before parents) through eval_node, no recursion. sm holds the query (q), its clauses (cl), nodes
// (nodes, n_nodes), phrase records (phrases) and the per-slot BM25 caches (cache[slot][norm byte]); phrase_posting(ix, sm, ...)
// is the engine's. A union slot that scores (a one-position multi-phrase) reads its entry's score (SmemUnions).
template <class Smem>
__device__ __forceinline__ bool eval_tree(const DevIndexView& ix, const Smem& sm, int32_t doc, uint64_t slot, float* out_score) {
  const uint32_t mask = presence_mask(slot);
  if ((mask & sm.q.req_term_mask) != sm.q.req_term_mask) return false;
  if (mask & sm.q.not_term_mask) return false;
  if (ix.live_bits && !((ix.live_bits[doc >> 5] >> (doc & 31)) & 1u)) return false;
  auto term = [&](const DevClause& c, float* s) {
    if (c.kind == NRTGPU_PHRASE) {
      if (c.col < 0) return false;   // a phrase of no terms
      const DevPhrase& ph = sm.phrases[c.col];
      for (int i = 0; i < ph.n_terms; ++i) if (!((mask >> sm.cl[ph.clause0 + i].slot) & 1u)) return false;
      const float f = phrase_freq(ix, sm, ph, doc, !c.scoring);
      if (f == 0.0f) return false;
      if (c.scoring) {
        const uint8_t* nrm = ix.norms[ph.field];
        const uint32_t nb = nrm ? (uint32_t)nrm[doc] : 1u;
        *s = bm25_score(c.weight, f, sm.cache[sm.cl[ph.clause0].slot][nb]);
      }
      return true;
    }
    const uint32_t b = (uint32_t)((slot >> (8 * c.slot)) & 0xff);
    if (b == 0) return false;
    if (c.scoring) {
      if constexpr (SmemUnions<Smem>::value) {
        if (c.plane == kUnionList) { *s = __ldg(sm.u.score + c.post_base + phrase_posting(ix, sm, c, doc)); return true; }
      }
      const float f = (b == 255u) ? exact_freq_slow(ix, c, doc) : (float)b;
      const uint8_t* nrm = ix.norms[c.field];
      const uint32_t nb = nrm ? (uint32_t)nrm[doc] : 1u;
      *s = bm25_score(c.weight, f, sm.cache[c.slot][nb]);
    }
    return true;
  };
  uint32_t matched = 0;
  float node_score[kMaxTreeNodes];
  for (int n = sm.n_nodes - 1; n >= 0; --n) {
    const DevNode& nd = sm.nodes[n];
    float s;
    if (!nd.empty && eval_node(ix, nd, sm.cl, doc, matched, node_score, term, &s)) { matched |= 1u << n; node_score[n] = s; }
  }
  if (!(matched & 1u)) return false;
  *out_score = node_score[0];
  return true;
}

}  // namespace nrtgpu
