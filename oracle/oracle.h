/*
 * oracle.h -- CPU restatement of the reference's query-execution arithmetic.
 *
 * TEST INFRASTRUCTURE ONLY. Nothing under nrtsearch_b200/ may include, link or
 * call this. Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs use it, as the checker / reported CPU baseline.
 *
 * The arithmetic lives in org.apache.lucene:lucene-core:10.4.0
 * (reference gradle/libs.versions.toml:7,42), which is NOT vendored in the
 * reference (Yelp/nrtsearch); it is restated here from Lucene's published algorithm and
 * anchored on the reference's own call sites and known-answer tests:
 *   - BM25 term score: pinned bit-exactly by
 *       src/test/java/com/yelp/nrtsearch/server/query/multifunction/MultiFunctionScoreQueryTest.java:139
 *       src/test/java/com/yelp/nrtsearch/server/grpc/SearchStateTest.java:117
 *       src/test/java/com/yelp/nrtsearch/server/grpc/QueryTest.java:1003-1018
 *       src/test/java/com/yelp/nrtsearch/server/similarity/SimilarityTest.java:114-120
 *     (tests/test_oracle_golden.py)
 *   - top-k order / search-after / thresholds: follows the in-tree
 *       src/main/java/org/apache/lucene/search/LazyQueueTopScoreDocCollector.java:103-144
 *   - vector score mapping: src/main/java/com/yelp/nrtsearch/server/field/VectorFieldDef.java:664-673,870-881
 *   - RRF blend: .../search/multiretriever/blender/score/WeightedRRFScoreDoc.java:60-77
 *   - rescore combine: src/main/java/com/yelp/nrtsearch/server/rescore/QueryRescore.java:39-46
 * PARITY UNPINNED (no reference test fixes them; stated from Lucene 10 behaviour):
 *   SmallFloat norms for length > 40, double summation of clause scores,
 *   ReqOptSumScorer's float add, TopDocs.merge tie-break, QueryRescorer re-sort.
 */
#ifndef NRT_ORACLE_H
#define NRT_ORACLE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- SmallFloat (Lucene org.apache.lucene.util.SmallFloat) ---- */
uint8_t orc_int_to_byte4(int32_t i);
int32_t orc_byte4_to_int(uint8_t b);

/* ---- BM25 (Lucene BM25Similarity; default chosen at
 *      src/main/java/com/yelp/nrtsearch/server/similarity/SimilarityCreator.java:33) ---- */
float orc_bm25_idf(int64_t doc_freq, int64_t doc_count);
float orc_bm25_avgdl(int64_t sum_total_term_freq, int64_t doc_count);
void  orc_bm25_cache(float k1, float b, float avgdl, float cache[256]);
float orc_bm25_score(float weight, float freq, uint8_t norm, const float cache[256]);

/* occur / kind codes shared with include/nrtgpu.h */
enum { ORC_SHOULD = 0, ORC_MUST = 1, ORC_FILTER = 2, ORC_MUST_NOT = 3 };
enum { ORC_TERM = 0, ORC_RANGE_I64 = 1, ORC_MATCH_ALL = 2 };

typedef struct {
  int32_t occur;   /* ORC_SHOULD.. */
  int32_t kind;    /* ORC_TERM.. */
  int32_t id;      /* term id (kind TERM) or doc-value column id (kind RANGE) */
  float   boost;   /* BoostQuery folded into the clause (weight = boost * idf) */
  int64_t lo, hi;  /* inclusive bounds for RANGE (sortable-int domain) */
} orc_clause;

typedef struct {
  int32_t clause_begin, clause_end;   /* into the clause array */
  int32_t min_should_match;
  int32_t has_after;                  /* search-after */
  int32_t after_doc; float after_score;
} orc_query;

typedef struct {
  int32_t n_docs;                    /* maxDoc of this shard; docs are 0..n_docs-1 locally */
  int32_t doc_base;                  /* added to local ids in results */
  int32_t n_terms;
  const int64_t* term_off;           /* [n_terms+1] CSR */
  const int32_t* post_docs;          /* local doc ids, ascending per term */
  const int32_t* post_freqs;
  const int32_t* term_field;         /* [n_terms] field id, or NULL = field 0 */
  const int64_t* term_df;            /* [n_terms] index-wide docFreq, or NULL = local CSR length */
  int32_t n_fields;
  const uint8_t* const* norms;       /* [n_fields] -> [n_docs] or NULL (omitNorms => norm byte 1) */
  const int64_t* field_doc_count;    /* [n_fields] index-wide */
  const int64_t* field_sum_ttf;      /* [n_fields] index-wide */
  const float* field_k1; const float* field_b;   /* [n_fields] or NULL => 1.2 / 0.75 */
  int32_t n_columns;
  const int64_t* const* columns;     /* [n_columns] -> [n_docs] int64 doc values (single valued) */
  const uint8_t* const* column_has;  /* [n_columns] -> [n_docs] 0/1 or NULL = all docs have a value */
  const uint8_t* live_docs;          /* [n_docs] 0/1 or NULL = all live */
  const float* term_max_x;           /* [n_terms] index-time impact max(freq*cache[norm]) or NULL */
  const int64_t* const* column_offsets; /* NULL, or [n_columns] -> int64[n_docs+1] for a MULTI-valued column (SORTED_NUMERIC):
                                          doc d holds columns[c][off[d] .. off[d+1]); NULL entry = single valued */
} orc_index;

/* fills term_max_x[n_terms] (index-time impacts; call once after the index arrays are set) */
void orc_build_term_max_x(const orc_index* ix, float* term_max_x);

/* mode 0: exhaustive (ScoreMode.COMPLETE); mode 1: dynamic pruning (MAXSCORE-style, TOP_SCORES).
 * Both return the same (doc, score) lists. total_hits is exact when relation==0 (EQUAL_TO).
 * out_docs/out_scores: [nq*top_k]; out_counts/out_total/out_rel: [nq]. Returns 0 or <0 on error. */
int orc_search(const orc_index* ix, const orc_clause* clauses, const orc_query* queries, int32_t nq,
               int32_t top_k, int32_t total_hits_threshold, int32_t mode, int32_t n_threads,
               int32_t* out_docs, float* out_scores, int32_t* out_counts, int64_t* out_total,
               uint8_t* out_rel);
/* sort-by-field top-k (TopFieldCollector semantics; reference SortFieldCollector.java:44-105, NumberFieldDef.java:266-278):
 * kind 1 = numeric doc-value column (values in the sortable-long domain), 2 = doc id; ties by doc asc; a doc without a
 * value sorts as missing_value; searchAfter = (after_values[q], queries[q].after_doc) when queries[q].has_after */
typedef struct { int32_t kind, column, reverse, reserved; int64_t missing_value; } orc_sort;
int orc_search_sorted(const orc_index* ix, const orc_clause* clauses, const orc_query* queries, int32_t nq, int32_t top_k,
                      int32_t n_threads, const orc_sort* sort, const int64_t* after_values, int32_t* out_docs,
                      int64_t* out_values, int32_t* out_counts, int64_t* out_total);

int orc_blend_scores(int32_t mode, int32_t n_retrievers, int32_t top_in, const int32_t* docs, const float* scores,
                     const int32_t* counts, const float* boosts, int32_t top_out, int32_t* out_docs, float* out_scores, int32_t* total);
int orc_match_bitmap(const orc_index* ix, const orc_clause* clauses, const orc_query* query, uint8_t* out_bitmap);
int orc_score_docs(const orc_index* ix, const orc_clause* clauses, const orc_query* queries, int32_t nq, int32_t n_hits,
                   const int32_t* docs, const int32_t* counts, uint8_t* out_matches, float* out_scores);

/* the same search under TerminateAfterWrapper (sequential semantics: docs in doc order; reference
 * src/main/java/com/yelp/nrtsearch/server/search/TerminateAfterWrapper.java:85-162): terminate_after 0 = none */
int orc_search_limits(const orc_index* ix, const orc_clause* clauses, const orc_query* queries, int32_t nq,
                      int32_t top_k, int32_t total_hits_threshold, int32_t mode, int32_t n_threads,
                      int32_t terminate_after, int32_t terminate_after_max_recall,
                      int32_t* out_docs, float* out_scores, int32_t* out_counts, int64_t* out_total,
                      uint8_t* out_rel, uint8_t* out_terminated);

/* TopDocs.merge(0, top_k, shards[]): inputs [n_lists][nq][top_k] sorted lists with counts [n_lists][nq]. */
void orc_merge_topk(int32_t n_lists, int32_t nq, int32_t top_k, const int32_t* docs, const float* scores,
                    const int32_t* counts, int32_t* out_docs, float* out_scores, int32_t* out_counts);

/* ---- vectors ---- */
enum { ORC_SIM_L2 = 0, ORC_SIM_DOT = 1, ORC_SIM_COSINE = 2, ORC_SIM_MIP = 3 };
/* raw similarity -> Lucene score (VectorSimilarityFunction.compare), float32 */
float orc_vector_score_f32(const float* a, const float* b, int32_t dims, int32_t sim);
/* exact brute force (ExactVectorQuery semantics): score*boost, top-k (score desc, doc asc) */
int orc_knn_exact(const float* corpus, int32_t n, int32_t dims, int32_t sim, int32_t doc_base,
                  const uint8_t* filter /*[n] 0/1 or NULL*/, const float* queries, int32_t nq,
                  const float* boosts /*[nq] or NULL*/, int32_t k, int32_t n_threads,
                  int32_t* out_docs, float* out_scores, int32_t* out_counts,
                  const uint8_t* live_docs /*[n] 0/1 or NULL: deleted docs are never hits*/);

/* ---- hybrid stages ---- */
/* weighted RRF over R retrievers; lists [R][top_in] with counts [R]; result sorted (score desc, doc asc);
 * returns number of hits written (<= top_out); *total = deduplicated count */
int orc_blend_rrf(int32_t n_retrievers, int32_t top_in, const int32_t* docs, const int32_t* counts,
                  const float* boosts, int32_t rank_constant, int32_t top_out, int32_t* out_docs,
                  float* out_scores, int32_t* total);
/* Lucene QueryRescorer.rescore + QueryRescore.combine: every hit combined, re-sorted
 * (score desc, doc asc) in place; the caller keeps the first `window` (= topN). */
void orc_rescore_combine(int32_t n_hits, int32_t window, int32_t* docs, float* scores,
                         const uint8_t* second_matches, const float* second_scores, double query_weight,
                         double rescore_weight);

#ifdef __cplusplus
}
#endif
#endif
