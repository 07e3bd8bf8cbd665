/*
 * nrtgpu.h -- C ABI of the H100-native query-execution engine that drops in behind nrtsearch's
 * SearchHandler / SearchRequestProcessor (reference = Yelp/nrtsearch @ 59c38655, Lucene 10.4.0).
 *
 * The reference has NO native seam for query execution (it is pure Java over lucene-core); the
 * entry points below are what a JNI shim would bind at the three Lucene API call sites that bound the
 * hot path (SURVEY.md section 8b):
 *
 *   nrtgpu_index_build / _close   <->  ShardSearcherFactory.newSearcher(reader, previous)
 *                                      src/main/java/com/yelp/nrtsearch/server/index/ShardState.java:506-526
 *                                      (one device image per reader version; freed after the last
 *                                      ShardState.release, :406-425)
 *   nrtgpu_search_bool            <->  searcher.search(query, collectorManager)
 *                                      src/main/java/com/yelp/nrtsearch/server/handler/SearchHandler.java:1412-1413, :556
 *                                      (BooleanQuery of TermQuery / range / match-all clauses built at
 *                                      .../query/QueryNodeMapper.java:257-283; collector config from
 *                                      .../search/collectors/RelevanceCollector.java:42-69)
 *   nrtgpu_search_knn             <->  knnQuery.rewrite(searcher)   .../search/KnnUtils.java:56
 *                                      and ExactVectorQuery          .../query/vector/ExactVectorQuery.java:137-173
 *   nrtgpu_merge_topk             <->  TopDocs.merge(0, numHits, perSlice[])
 *                                      src/main/java/org/apache/lucene/search/LazyQueueTopScoreDocCollectorManager.java:137-144
 *   nrtgpu_blend_rrf              <->  BlenderOperation.blend (weighted RRF)
 *                                      .../search/multiretriever/blender/BlenderOperation.java:76-87
 *   nrtgpu_rescore_combine        <->  RescoreOperation.rescore / QueryRescore.combine
 *                                      .../rescore/QueryRescore.java:39-57
 *
 * Conventions: every function returns 0 on success, non-zero nrtgpu_status otherwise; the message is
 * available from nrtgpu_last_error() (thread-local). Handles are opaque; output buffers are caller
 * allocated (Java direct ByteBuffers); the library never frees caller memory. All entry points are
 * re-entrant (called concurrently from the reference's SERVER / SEARCH / RETRIEVER pools).
 * There is NO CPU fallback: without a CUDA device every call fails with NRTGPU_ERR_CUDA.
 */
#ifndef NRTGPU_H
#define NRTGPU_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  NRTGPU_OK = 0,
  NRTGPU_ERR_INVALID = 1,      /* IllegalArgumentException on the Java side */
  NRTGPU_ERR_CUDA = 2,         /* -> Status.INTERNAL (SearchHandler.java:136-145) */
  NRTGPU_ERR_UNSUPPORTED = 3,  /* query shape outside the GPU path: caller falls through to Lucene */
  NRTGPU_ERR_OOM = 4,
  NRTGPU_ERR_TIMEOUT = 5       /* CollectionTimeoutException (SearchCutoffWrapper.java:164-174, noPartialResults) */
} nrtgpu_status;

typedef struct nrtgpu_ctx nrtgpu_ctx;     /* one per (process, device) */
typedef struct nrtgpu_index nrtgpu_index; /* device image of one shard at one reader version */
typedef struct nrtgpu_batch nrtgpu_batch; /* a compiled query batch resident on the device */

const char* nrtgpu_last_error(void);
int nrtgpu_version(void);

/* device_id: CUDA ordinal (one shard group per GPU; one process per GPU). */
int nrtgpu_init(int device_id, nrtgpu_ctx** out);
void nrtgpu_shutdown(nrtgpu_ctx* ctx);

/* BooleanClause.Occur and leaf kinds */
enum { NRTGPU_SHOULD = 0, NRTGPU_MUST = 1, NRTGPU_FILTER = 2, NRTGPU_MUST_NOT = 3 };
enum { NRTGPU_TERM = 0, NRTGPU_RANGE_I64 = 1, NRTGPU_MATCH_ALL = 2 };
/* VectorSimilarityFunction (reference VectorFieldDef.java:77-88) */
enum { NRTGPU_SIM_L2 = 0, NRTGPU_SIM_DOT = 1, NRTGPU_SIM_COSINE = 2, NRTGPU_SIM_MIP = 3 };
enum { NRTGPU_VEC_FLOAT32 = 0, NRTGPU_VEC_INT8 = 1 };

/* Host-side description of one shard, i.e. what the adaptor reads out of the LeafReaders
 * (terms()/postings()/getNormValues()/getNumericDocValues()/getFloatVectorValues()). Term ids are the
 * adaptor's dense numbering of (field, term); doc ids are shard-local, results carry doc_base + local. */
typedef struct {
  int32_t n_docs;
  int32_t doc_base;
  int32_t n_terms;
  const int64_t* term_off;          /* [n_terms+1] CSR offsets into post_* */
  const int32_t* post_docs;         /* ascending per term */
  const int32_t* post_freqs;        /* >= 1 */
  const int32_t* term_field;        /* [n_terms] text-field id, NULL = all field 0 */
  const int64_t* term_df;           /* [n_terms] INDEX-WIDE docFreq (termStatistics), NULL = CSR length */
  int32_t n_fields;
  const uint8_t* const* norms;      /* [n_fields] -> [n_docs] SmallFloat norm bytes, NULL entry = omitNorms */
  const int64_t* field_doc_count;   /* [n_fields] INDEX-WIDE collectionStatistics.docCount */
  const int64_t* field_sum_ttf;     /* [n_fields] INDEX-WIDE sumTotalTermFreq */
  const float* field_k1;            /* [n_fields] or NULL => 1.2 */
  const float* field_b;             /* [n_fields] or NULL => 0.75 */
  int32_t n_columns;
  const int64_t* const* columns;    /* [n_columns] -> [n_docs] numeric doc values (sortable-long domain) */
  const uint8_t* const* column_has; /* [n_columns] -> [n_docs] 0/1, NULL entry = every doc has a value */
  const uint8_t* live_docs;         /* [n_docs] 0/1 or NULL */
  /* one float vector field (more via nrtgpu_index_add_vectors) */
  int32_t vec_dims;                 /* 0 = none */
  int32_t vec_similarity;
  int32_t vec_count;                /* number of vectors (ord -> doc via vec_docs, NULL = identity) */
  const float* vectors;             /* [vec_count * vec_dims] float32, or int8 when vec_element_type == NRTGPU_VEC_INT8 */
  const int32_t* vec_docs;
  int32_t vec_element_type;         /* NRTGPU_VEC_FLOAT32 (FloatVectorFieldDef) or NRTGPU_VEC_INT8 (ByteVectorFieldDef: scores by
                                       VectorFieldDef.java:870-881, i.e. DOT_PRODUCT = 0.5 + dot / (dims * 2^15); queries are passed
                                       as floats holding the byte values) */
  const int64_t* const* column_offsets; /* NULL, or [n_columns]: a non-NULL entry makes column c MULTI-valued (SORTED_NUMERIC doc
                                       values, reference NumberFieldDef.java multiValued): int64[n_docs+1] offsets into columns[c],
                                       which then holds the flattened values, ascending within a doc. A range clause matches a doc
                                       when ANY of its values lies in [lo, hi] (SortedNumericDocValuesRangeQuery; keyword
                                       columns take NRTGPU_KEYWORD_RANGE clauses with the same rule). nrtgpu_search_sorted,
                                       terms / min / max / sum collectors and fetch on such a column answer NRTGPU_ERR_UNSUPPORTED;
                                       nrtgpu_search_sorted_fields sorts on it (MIN / MAX selector). */
} nrtgpu_shard_desc;

int nrtgpu_index_build(nrtgpu_ctx* ctx, const nrtgpu_shard_desc* desc, nrtgpu_index** out);
int nrtgpu_index_close(nrtgpu_index* ix);
/* bytes of device memory held by the image */
int64_t nrtgpu_index_device_bytes(const nrtgpu_index* ix);

typedef struct {
  int32_t occur;  /* NRTGPU_SHOULD.. */
  int32_t kind;   /* NRTGPU_TERM.. */
  int32_t id;     /* term id or column id */
  float boost;    /* product of enclosing BoostQuery boosts (weight = boost * idf). Every entry point that compiles
                     clauses refuses, with NRTGPU_ERR_INVALID and no output written, a boost < 0 ("Boost must be a
                     positive number", QueryNodeMapper.java:127) and a NaN or infinite one ("Boost must be a finite
                     number", as Lucene's BoostQuery refuses it). 0 is a weight of 0. */
  int64_t lo, hi; /* inclusive range bounds */
} nrtgpu_clause;

typedef struct {
  int32_t clause_begin, clause_end; /* flat BooleanQuery = clauses[clause_begin:clause_end] */
  int32_t min_should_match;
  int32_t has_after;                /* searchAfter (LazyQueueTopScoreDocCollector.java:112) */
  int32_t after_doc;
  float after_score;
} nrtgpu_query;

/* flags */
enum {
  NRTGPU_FLAG_NONE = 0,
  NRTGPU_FLAG_NO_PRUNING = 1     /* force exhaustive evaluation (exact totalHits) even when total_hits_threshold < MAX
                                    would allow MAXSCORE: by default, once a query has collected more than
                                    total_hits_threshold hits, lists whose score bounds cannot reach the running k-th
                                    score stop driving the sweep -- same (doc, score) lists, totalHits becomes a lower
                                    bound (relation 1), exactly the contract of the reference's TOP_SCORES mode */
};

/* One-shot search with HOST buffers (the JNI entry point): uploads the batch, runs, copies results
 * back, synchronises `stream` (a cudaStream_t, NULL = default stream).
 *   out_docs/out_scores [nq*top_k] (score desc, doc asc), out_counts [nq],
 *   out_total_hits [nq], out_relation [nq] (0 = EQUAL_TO, 1 = GREATER_THAN_OR_EQUAL_TO).
 * total_hits_threshold == INT32_MAX <=> ScoreMode.COMPLETE (exact counts, no pruning). */
int nrtgpu_search_bool(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                       const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                       int32_t total_hits_threshold, int32_t flags, void* stream, int32_t* out_docs,
                       float* out_scores, int32_t* out_counts, int64_t* out_total_hits,
                       uint8_t* out_relation);

/* Deadline and terminateAfter of a search (DocCollector config: timeoutSec, terminateAfter, terminateAfterMaxRecallCount,
 * disallowPartialResults -- reference src/main/java/com/yelp/nrtsearch/server/search/collectors/CollectorCreatorContext.java:36-53,
 * wrappers SearchCutoffWrapper.java:164-202 and TerminateAfterWrapper.java:85-162).
 *  - timeout_sec > 0: the timer starts when the first work item of the batch starts on the device (elapsed_sec = time the
 *    request already spent before the call is subtracted); it is checked at every work-item boundary ((query, <= 512K-doc
 *    slice): the reference checks per segment and, optionally, every timeoutCheckEvery docs). Work items claimed after the
 *    deadline are skipped: the query returns the hits collected so far with out_hit_timeout = 1 and relation GTE, or, with
 *    disallow_partial_results, the call fails with NRTGPU_ERR_TIMEOUT ("Search collection exceeded timeout of ...s").
 *  - terminate_after > 0: a query that has collected that many hits takes no further work items; whenever more than
 *    terminate_after docs match, out_terminated_early = 1, relation GTE and totalHits = hits counted, capped at
 *    terminate_after_max_recall_count. (The reference's slices race on one AtomicInteger, so WHICH docs are collected
 *    before the cut is timing dependent there too; here the cut falls on work-item boundaries.)
 * Both apply to queries the posting-probe kernel runs (<= 4 term clauses led by a posting list); others ignore them. */
typedef struct {
  double timeout_sec;                       /* 0: none */
  double elapsed_sec;                       /* already spent by the request before this call */
  int32_t disallow_partial_results;
  int32_t terminate_after;                  /* 0: none */
  int32_t terminate_after_max_recall_count; /* 0: = terminate_after */
} nrtgpu_search_limits;

/* nrtgpu_search_bool + limits; out_hit_timeout / out_terminated_early [nq] may be NULL */
int nrtgpu_search_bool_ex(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                          const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                          int32_t total_hits_threshold, int32_t flags, const nrtgpu_search_limits* limits,
                          void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                          int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout,
                          uint8_t* out_terminated_early);
/* Query trees (BooleanQuery and DisjunctionMaxQuery nested in a BooleanQuery, reference QueryNodeMapper.java:257-283 for
 * bool, :360-395 for a match of several tokens, :429-497 for multi_match BEST_FIELDS). The leaves are the clause kinds
 * above; a clause of kind NRTGPU_NODE is a nested query whose id indexes nodes[], and each node's clauses are
 * clauses[clause_begin:clause_end] of the same array. The root of query q is still queries[q] (a BooleanQuery with its
 * msm and searchAfter); a DisjunctionMaxQuery at the root is a root with one MUST node clause, and scores exactly as the
 * dismax does.
 *   BOOL node:   the rule of a flat BooleanQuery, a child node counting as a clause that scores the child's float;
 *   DISMAX node: matches if any disjunct does, scores (float)((double)max + others * (double)tie_breaker), where others is
 *                the double sum of the other matching disjuncts (DisjunctionMaxScorer, Lucene 10).
 *   CONSTANT node (ConstantScoreQuery; ExistsQuery is one over the term of its field in the _field_names field): matches
 *                when its clause does and scores its boost; nothing below it scores (a phrase stops at its first match);
 *   MIN_SCORE node (MinScoreQuery, the reference's MinThresholdQuery): its clause is scored with boost 1 below the node
 *                (boosts below it still fold into its leaves) and always scores, even under FILTER, MUST_NOT or CONSTANT;
 *                with s its float score the node matches iff s >= min_score in float (a NaN threshold matches nothing)
 *                and scores __fmul_rn(s, boost). A threshold of 0 is an ordinary threshold here: the reference returns
 *                the inner query unwrapped at 0, boosts folded into its leaves, which the caller compiles as that query.
 *                Both kinds hold exactly one clause, whose occur is MUST (any leaf kind or a node clause). Their boost
 *                is the float product, outermost first, of the BoostQuerys above the node.
 * Subtrees under FILTER, MUST_NOT and CONSTANT only match, unless a MIN_SCORE node below scores its own. Boosts are
 * folded into the leaves (outermost first, in float), stopping at a CONSTANT or MIN_SCORE node, which takes them as its
 * boost: a node clause has boost 1. A CONSTANT or MIN_SCORE query at the root is a root with one MUST node clause.
 * Every tree batch runs on the window engine (as a batch with more than 4 term clauses does).
 *   NRTGPU_ERR_INVALID:     a node id out of range, a node referenced twice or from a cycle, a bad node kind or clause
 *                           range, a DISMAX clause whose occur is not SHOULD, tie_breaker outside [0, 1], a node clause
 *                           whose boost is not 1, msm < 0, a CONSTANT or MIN_SCORE node without exactly one clause or
 *                           whose clause is not MUST, a CONSTANT or MIN_SCORE boost < 0, NaN or infinite, a min_score < 0
 *                           ("MinScoreQuery.min_score must be a non-negative number"), and every check of
 *                           nrtgpu_search_bool_ex.
 *   NRTGPU_ERR_UNSUPPORTED: more than 8 term leaves, 8 nodes or 32 clauses in one tree, more than 4 levels of queries
 *                           (the root counts as one), top_k > 1024. CONSTANT and MIN_SCORE nodes count as nodes and
 *                           levels, their clause as a clause.
 * With n_nodes == 0 nrtgpu_search_tree is nrtgpu_search_bool_ex (same compile, same engine); the other entry points
 * reject NRTGPU_NODE clauses as a bad clause kind. Node kinds 2 and 5 are not kinds.
 *
 * NESTED node (NestedQuery, reference QueryNodeMapper.getNestedQuery: Lucene 10 ToParentBlockJoinQuery): a block join.
 * The image stores each parent as a block, its child docs first and the parent last; the parents are the docs of one
 * term (nrtgpu_index_add_parents, the _nested_path:_root term). The node holds exactly one MUST clause, the child query,
 * which the caller builds as the reference does: a BOOL node {FILTER _nested_path:<path>, MUST child}. min_should_match
 * holds the score mode (the proto's NestedQuery.ScoreMode): NONE 0, AVG 1, MAX 2, MIN 3, SUM 4; tie_breaker, boost and
 * min_score are not read. The child query is evaluated WITHOUT live docs (the child scorer does not read acceptDocs); a
 * matching child c joins the smallest parent doc > c, and joins nothing when it is itself a parent or follows the image's
 * last parent. A parent with n >= 1 joined children of float scores s_1..s_n (child doc order) matches and scores
 *   NONE: 0.0f;  SUM: (float) of the double sum in child order;  AVG: (float)(double sum / n);  MAX / MIN: the largest /
 *   smallest s_i,
 * and is then a hit as any doc is (its own liveness applies). Boosts above the node fold through it into the child query's
 * leaves; the node has no boost of its own. Under FILTER, MUST_NOT or CONSTANT, or with NONE, the child query only has to
 * match (a MIN_SCORE node inside it still scores its own subtree). Joins may appear at any depth and under every occur,
 * but not inside a child query. Each join is built on the device by the call (once by a prepared batch): the child query
 * runs over every slice, its matches are sorted and folded into one (parent, score) list per join, and the parent query
 * reads that list as a term slot. Like the multi-phrase unions' build, this runs when the batch is built and does not
 * check the search deadline, and the child matches count toward no totalHits or terminateAfter.
 * Limits: the tree limits (8 term slots, 8 nodes, 32 clauses, 4 levels) apply to the parent tree, where each join takes
 * one term slot and one clause, and separately to each child tree, rooted at the join's clause. Before any launch, each
 * join's child matches are bounded by the postings of its child query's driver lists (a multi-phrase union slot at its
 * gathered postings; a query without a driver list at the image's doc count); a call whose bounds sum to more than 2^26
 * is refused. The join scratch takes 40 bytes per bounded child (sort keys and scores, double-buffered; run heads and
 * their scan; the entries behind the union entries), plus the sort's temporary storage. It belongs to the batch that runs the call and, like the union scratch, only grows.
 * NRTGPU_JOIN_CHILDREN, read when the context is created, lowers the cap (> 0).
 *   NRTGPU_ERR_INVALID:     a NESTED node without exactly one clause or whose clause is not MUST, a score mode outside
 *                           0..4, an image without parents ("index has no parent docs: nrtgpu_index_add_parents");
 *   NRTGPU_ERR_UNSUPPORTED: a NESTED node inside a join's child query, the join cap, a tree limit of the parent tree or
 *                           of a child tree.
 * A refused call writes no output and launches nothing. Accepted by nrtgpu_search_tree, nrtgpu_search_tree_phrases,
 * nrtgpu_batch_prepare_tree[_phrases], nrtgpu_search_tree_aggs, nrtgpu_searcher_search_tree_phrases and
 * nrtgpu_searcher_search_tree_aggs (every leaf with its own parents: blocks never straddle leaves); tree rescoring
 * (nrtgpu_score_docs_tree, nrtgpu_rescore_query_tree) answers "bad node kind". */
enum { NRTGPU_NODE = 3 };
enum { NRTGPU_NODE_BOOL = 0, NRTGPU_NODE_DISMAX = 1, NRTGPU_NODE_CONSTANT = 3, NRTGPU_NODE_MIN_SCORE = 4,
       NRTGPU_NODE_NESTED = 6 };
enum { NRTGPU_NESTED_NONE = 0, NRTGPU_NESTED_AVG = 1, NRTGPU_NESTED_MAX = 2, NRTGPU_NESTED_MIN = 3, NRTGPU_NESTED_SUM = 4 };
typedef struct {
  int32_t kind;                      /* NRTGPU_NODE_BOOL / _DISMAX / _CONSTANT / _MIN_SCORE / _NESTED */
  int32_t clause_begin, clause_end;  /* its clauses in the same clauses[] array */
  int32_t min_should_match;          /* BOOL; NESTED: the score mode */
  float tie_breaker;                 /* DISMAX: tieBreakerMultiplier, in [0, 1] */
  float boost;                       /* CONSTANT / MIN_SCORE (BOOL and DISMAX do not read it) */
  float min_score;                   /* MIN_SCORE: the threshold, >= 0 or NaN */
} nrtgpu_node;
int nrtgpu_search_tree(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                       int32_t n_nodes, const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                       int32_t total_hits_threshold, int32_t flags, const nrtgpu_search_limits* limits, void* stream,
                       int32_t* out_docs, float* out_scores, int32_t* out_counts, int64_t* out_total_hits,
                       uint8_t* out_relation, uint8_t* out_hit_timeout, uint8_t* out_terminated_early);
/* split form of nrtgpu_search_tree: then nrtgpu_batch_run / _fetch / _bind_packed / ... as for nrtgpu_batch_prepare */
int nrtgpu_batch_prepare_tree(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                              int32_t n_nodes, const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                              int32_t total_hits_threshold, int32_t flags, nrtgpu_batch** out);

/* Term positions of an image (PostingsEnum.nextPosition() with PostingsEnum.POSITIONS): positions[] holds, posting after
 * posting in the CSR order of the build, the freq positions of that posting, ascending (equal positions are allowed);
 * n_positions must be the sum of the build's freqs. A second call replaces the positions. They stay valid across
 * nrtgpu_index_set_live_docs and nrtgpu_index_update_stats, and nrtgpu_index_device_bytes counts them (4 B per position,
 * 4 B per posting and 8 B per term). NRTGPU_ERR_INVALID: a wrong count, a negative position, positions that descend
 * within a posting. */
int nrtgpu_index_add_positions(nrtgpu_index* ix, const int32_t* positions, int64_t n_positions);

/* The parent docs of an image's blocks (NRTGPU_NODE_NESTED): the docs of term root_term (the _nested_path:_root term,
 * QueryBitSetProducer of the reference's IndexState), as a bitset on the device (N / 8 bytes, counted by
 * nrtgpu_index_device_bytes). It stays valid across nrtgpu_index_set_live_docs and nrtgpu_index_update_stats; a second
 * call replaces it. NRTGPU_ERR_INVALID: a term out of range. */
int nrtgpu_index_add_parents(nrtgpu_index* ix, int32_t root_term);

/* Keyword columns of an image (string doc values of atom / text-with-docValues fields: SortedDocValues and
 * SortedSetDocValues of the leaf). Column k of the call is keyword column k of the image; terms aggregations name it with
 * value_type NRTGPU_AGG_VALUE_KEYWORD, keyword sorts, NRTGPU_KEYWORD_RANGE clauses and NRTGPU_AGG_FILTER_KEYWORD_SET
 * filters by its index. Per column:
 *   term_bytes / term_offsets [n_terms + 1]  the leaf's term dictionary, term i = term_bytes[term_offsets[i], term_offsets[i + 1]),
 *            strictly ascending in unsigned-byte order (BytesRef.compareTo); ordinal i is term i;
 *   multi_valued 0 (SORTED)      ords [n_docs]: the doc's ordinal, -1: no value;
 *   multi_valued 1 (SORTED_SET)  doc_offsets [n_docs + 1] (doc_offsets[0] == 0, non-decreasing) and ords [doc_offsets[n_docs]]:
 *            the doc's ordinals strictly ascending (SortedSetDocValues has each term of a doc once).
 * On the device an ordinal i is the bucket code 2i + 2 (0: no value): 4 B per doc (SORTED), or 4 B per value plus the
 * int64 doc offsets (SORTED_SET). The dictionary stays on the host (bucket keys, reader-wide dictionaries).
 * nrtgpu_index_device_bytes counts the device arrays. The columns stay valid across nrtgpu_index_set_live_docs and
 * nrtgpu_index_update_stats.
 *   NRTGPU_ERR_INVALID (the image is left unchanged): n < 0, a NULL array, a bad multi_valued, n_terms < 0, term offsets that
 *     do not start at 0 or descend, terms that are not strictly ascending (unsorted or duplicate), an ordinal outside
 *     [0, n_terms) (SORTED: -1 allowed), doc offsets that do not start at 0 or descend, ordinals of a doc that do not strictly
 *     ascend, and a second call on the image. */
typedef struct {
  int32_t n_terms;
  int32_t multi_valued;          /* 0: SORTED, 1: SORTED_SET */
  const uint8_t* term_bytes;
  const int64_t* term_offsets;   /* [n_terms + 1] */
  const int32_t* ords;           /* SORTED: [n_docs]; SORTED_SET: [doc_offsets[n_docs]] */
  const int64_t* doc_offsets;    /* SORTED_SET: [n_docs + 1]; SORTED: unused */
} nrtgpu_keyword_column;
int nrtgpu_index_add_keyword_columns(nrtgpu_index* ix, const nrtgpu_keyword_column* cols, int32_t n);
/* The bytes of term `ord` of keyword column `column` of an image: its length in *len, and its first min(len, cap) bytes
 * in out (out may be NULL when cap is 0). NRTGPU_ERR_INVALID: a column or ordinal out of range, len NULL. */
int nrtgpu_index_keyword_term(const nrtgpu_index* ix, int32_t column, int32_t ord, uint8_t* out, int32_t cap, int32_t* len);
/* The sort code of a term (bytes[0 .. len)) in keyword column `column` of an image (NRTGPU_SORT_KEYWORD values): 2i + 2
 * when the dictionary holds it as term i, else 2i + 1 where i is the number of terms that sort before it (unsigned-byte
 * order). A searchAfter term from LastHitInfo becomes an after value this way. NRTGPU_ERR_INVALID: a column out of range,
 * code NULL, bytes NULL with len > 0, len < 0. */
int nrtgpu_index_keyword_seek(const nrtgpu_index* ix, int32_t column, const uint8_t* bytes, int32_t len, int64_t* code);

/* Keyword range clauses (TermRangeQuery and SortedSetDocValuesField.newSlowRangeQuery on an atom field, AtomFieldDef.getRangeQuery;
 * PrefixQuery on an atom field with a constant-score rewrite, AtomFieldDef.getPrefixQuery). A clause of kind
 * NRTGPU_KEYWORD_RANGE tests keyword column `id` (nrtgpu_index_add_keyword_columns) against the inclusive code range
 * [lo, hi]: codes of the image's dictionary on an image, of the reader-wide union on a searcher (as keyword sort values).
 * Ordinals follow unsigned-byte term order, so the terms a range or a prefix matches are one run of codes. A SORTED doc
 * matches when its code is in [lo, hi], a SORTED_SET doc when any of its codes is; a doc without a value never matches.
 * The clause is constant-score (score = boost) under every occur, exactly as NRTGPU_RANGE_I64, and every entry point that
 * takes a range clause takes it (flat and tree batches, sorted search, collectors and their filter queries, kNN filter
 * queries, the second pass, the micro-batcher). lo > hi is an empty range and matches no doc.
 *   NRTGPU_ERR_INVALID: "keyword column out of range" (an image without keyword columns included), "keyword code out of
 *   range" for lo or hi outside [1, 2n + 1] (n: the dictionary's terms).
 * nrtgpu_index_keyword_range / nrtgpu_searcher_keyword_range turn term bounds into that range. With c = the
 * nrtgpu_index_keyword_seek code of a bound (2i + 2 for a held term, 2i + 1 for the gap before term i):
 *   lower inclusive lo = c, exclusive lo = c + 1 when c is even (else c), NO_LOWER lo = 1;
 *   upper inclusive hi = c, exclusive hi = c - 1 when c is even (else c), NO_UPPER hi = 2n + 1;
 *   PREFIX: lower is the prefix p (upper is unused): lo = seek(p), and the upper bound is succ(p) exclusive, where succ(p) is
 *   p with its trailing 0xFF bytes dropped and its last byte incremented; an empty or all-0xFF prefix has no upper bound.
 * The bounds are bytes as the field indexes them: applying the field's normalizer is the caller's. NRTGPU_ERR_INVALID: a
 * keyword column out of range, lo or hi NULL, a bound NULL with a length > 0, a negative length, a bad flag. */
enum { NRTGPU_KEYWORD_RANGE = 5 };
enum { NRTGPU_KEYWORD_NO_LOWER = 1, NRTGPU_KEYWORD_NO_UPPER = 2, NRTGPU_KEYWORD_LOWER_EXCLUSIVE = 4,
       NRTGPU_KEYWORD_UPPER_EXCLUSIVE = 8, NRTGPU_KEYWORD_PREFIX = 16 };
int nrtgpu_index_keyword_range(const nrtgpu_index* ix, int32_t column, const uint8_t* lower, int32_t lower_len,
                               const uint8_t* upper, int32_t upper_len, int32_t flags, int64_t* lo, int64_t* hi);

/* Phrase leaves of query trees (PhraseQuery / match_phrase, reference QueryNodeMapper.java:285-291, :397-427). A clause of
 * kind NRTGPU_PHRASE is a leaf whose id indexes phrases[]; its boost is the leaf's folded boost, as for a term leaf. The
 * phrase's terms are phrase_terms[term_begin:term_end] with their PhraseQuery positions (PhraseQuery.getTerms() /
 * getPositions()); slop is PhraseQuery.getSlop(). Lucene 10 PhraseWeight semantics:
 *   weight:  boost * idf, idf = (float) of the double sum of every term's float idf, a repeated term counted each time
 *            (BM25Similarity.idfExplain over the term statistics); score = BM25(weight, freq, norm of the phrase's field);
 *   slop 0:  ExactPhraseMatcher. The lead is the term of the smallest position (the first one given on a tie); freq is the
 *            number of the lead's positions p in the doc (each occurrence counted) at which every other term i has a
 *            position p - position_lead + position_i. Overlapping occurrences count ("a a" in "a a a" has freq 2);
 *   slop>0:  SloppyPhraseMatcher without repeats: a queue of (doc position - query position, query position, ordinal) per
 *            term, the running end and the match-length minimisation; every match of matchLength <= slop adds
 *            1.0f / (1.0f + matchLength) to freq, in float, in the matcher's order;
 *   a phrase of no terms matches nothing, one of one term is that term's leaf (Lucene's rewrite). Under FILTER and
 *   MUST_NOT a phrase only has to match. Phrase terms take term slots: a tree holds at most 8 term leaves and phrase
 *   terms together. Phrases run on the window engine only.
 *   NRTGPU_ERR_INVALID:     a phrase id or phrase term id out of range, a term range out of bounds, terms of different
 *                           fields, negative or descending positions, slop < 0, an image without positions
 *                           (nrtgpu_index_add_positions: "field was indexed without position data"), every check of
 *                           nrtgpu_search_tree;
 *   NRTGPU_ERR_UNSUPPORTED: more than 8 term slots in one tree, a sloppy phrase with a repeated term (Lucene's repeat
 *                           groups), every limit of nrtgpu_search_tree.
 * With n_phrases == 0 these are nrtgpu_search_tree / nrtgpu_batch_prepare_tree. A batch holding a phrase is a tree batch
 * even without nodes (a bare PhraseQuery is a root with one MUST phrase clause). Every other entry point rejects
 * NRTGPU_PHRASE clauses as a bad clause kind.
 *
 * Multi-phrase leaves (MultiPhraseQuery: match_phrase_prefix, multi_match PHRASE_PREFIX, match_phrase over stacked
 * synonyms). A clause of kind NRTGPU_MULTI_PHRASE is a leaf whose id indexes phrases[] as for NRTGPU_PHRASE; its
 * phrase_terms share positions (given in non-decreasing order), and terms that share a position are ALTERNATIVES: a doc
 * matches a position when any of them occurs there. The positions of a position are the merged positions of its terms,
 * repeats kept (UnionPostingsEnum). Prefix expansion is the caller's: it passes the expanded terms' ids. Semantics:
 *   weight:  boost * (float) of the double sum of the float idf of every term with df > 0 over all positions, a term
 *            repeated at several positions counted each time (MultiPhraseQuery.createWeight), summed position after
 *            position, ascending term id within one; no such term: the leaf matches nothing. Score as for NRTGPU_PHRASE; slop 0
 *            is ExactPhraseMatcher over the merged positions, slop > 0 SloppyPhraseMatcher;
 *   one position (MultiPhraseQuery.rewrite): a BooleanQuery of SHOULD TermQuerys over its alternatives: matches a doc
 *            holding any of them and scores (float) of the double sum of each present alternative's BM25 at weight
 *            boost * idf of that term, summed in ascending term id order (one alternative: that TermQuery);
 *   no positions: matches nothing. Under FILTER, MUST_NOT and inside a CONSTANT node it only has to match.
 * Limits: every position takes ONE term slot, however many alternatives it has (<= 8 slots per tree, term leaves,
 * phrase terms and multi-phrase positions together); at most 128 alternatives per position; per call the distinct
 * alternative sets of a position (deduplicated over the batch's queries; a one-position leaf's set is keyed by its
 * boost too) gather at most 2^25 postings (52 bytes of device scratch each, 1.75 GB) and merge at most 2^27
 * positions (4 bytes each, 512 MB). The unions are built on the device by each call (and once by a prepared batch). The
 * scratch belongs to the batch that runs the call (an index's reused search workspace for the one-shot calls) and, like
 * that batch's other buffers, only grows: after a call near the caps up to 2.25 GB stay allocated until the index (or the
 * prepared batch) is freed. NRTGPU_UNION_POSTINGS, read when the context is created, lowers the postings cap (> 0).
 *   NRTGPU_ERR_INVALID:     as for NRTGPU_PHRASE (an image without positions only with two or more positions);
 *   NRTGPU_ERR_UNSUPPORTED: more than 8 term slots, more than 128 terms at one position, a sloppy multi-phrase in
 *                           which one term appears at two positions, the union postings or positions cap.
 * A refused call writes no output. Accepted by nrtgpu_search_tree_phrases, nrtgpu_batch_prepare_tree_phrases,
 * nrtgpu_search_tree_aggs, nrtgpu_searcher_search_tree_phrases and nrtgpu_searcher_search_tree_aggs; every other entry
 * point, tree rescoring (nrtgpu_score_docs_tree, nrtgpu_rescore_query_tree) included, rejects it as a bad clause kind. */
enum { NRTGPU_PHRASE = 4, NRTGPU_MULTI_PHRASE = 6 };
typedef struct { int32_t term_begin, term_end; int32_t slop; int32_t reserved; } nrtgpu_phrase;
typedef struct { int32_t term; int32_t position; } nrtgpu_phrase_term;
int nrtgpu_search_tree_phrases(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                               int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                               const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                               int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags,
                               const nrtgpu_search_limits* limits, void* stream, int32_t* out_docs, float* out_scores,
                               int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout,
                               uint8_t* out_terminated_early);
int nrtgpu_batch_prepare_tree_phrases(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                                      const nrtgpu_node* nodes, int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                                      const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms,
                                      const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t total_hits_threshold,
                                      int32_t flags, nrtgpu_batch** out);

/* same search with HOST query buffers, results left on the DEVICE in one packed record (see nrtgpu_packed_words): the
 * multi-GPU request path (the caller all-gathers the record on `stream`, then nrtgpu_merge_topk_packed). Synchronises. */
int nrtgpu_search_bool_packed(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                              const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                              int32_t total_hits_threshold, int32_t flags, const nrtgpu_search_limits* limits,
                              void* stream, int32_t* d_record);

/* Sort-by-field top-k (TopFieldCollector; reference src/main/java/com/yelp/nrtsearch/server/search/collectors/
 * SortFieldCollector.java:44-105, sort construction .../search/sort/SortParser.java:54-131, numeric sort fields
 * .../field/NumberFieldDef.java:266-278 = SortedNumericSortField(type, reverse) with missingValue from
 * getSortMissingValue(missingLast)). One sort key + the implicit doc-id tie-break (lower doc first), i.e. the Sort
 * [<numeric doc-value field>], [docid] or [docid reverse]; other sorts (several fields, score mixed in) return
 * NRTGPU_ERR_UNSUPPORTED (nrtgpu_search_sorted_fields below serves them). Values live in the column's sortable-long domain (the adaptor maps int/long directly and
 * float/double through NumericUtils.floatToSortableInt / doubleToSortableLong, exactly as the range query bounds).
 *   missing_value: what a doc WITHOUT a value sorts as (Integer/Long.MIN|MAX_VALUE, -+Infinity in the sortable domain:
 *                  the reference picks MAX when missingLast, irrespective of `reverse`);
 *   after_values:  per query, the sort value of the last hit of the previous page (FieldDoc.fields[0]); used with
 *                  nrtgpu_query.has_after / after_doc (LastHitInfo, SortParser.parseLastHitInfo :131-160). A hit
 *                  qualifies iff its value sorts strictly after the after value, or ties with it and has a greater
 *                  global doc id than after_doc; the value need not be held by any doc of this leaf. A doc without a
 *                  value sorts as missing_value whether or not any doc holds that value: it ties with an after value
 *                  equal to missing_value, and is compared by value with any other after value.
 * Results: docs in sort order, out_sort_values = the FieldDoc value of every hit (missing docs carry missing_value),
 * scores are NaN (TopFieldCollector does not track scores), totalHits exact (relation EQUAL_TO). */
enum { NRTGPU_SORT_RELEVANCE = 0, NRTGPU_SORT_COLUMN = 1, NRTGPU_SORT_DOCID = 2 };
typedef struct {
  int32_t kind;          /* NRTGPU_SORT_* */
  int32_t column;        /* NRTGPU_SORT_COLUMN: doc-value column id */
  int32_t reverse;       /* SortType.reverse */
  int32_t reserved;
  int64_t missing_value;
  const int64_t* after_values; /* [nq] or NULL */
} nrtgpu_sort;

int nrtgpu_search_sorted(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                         const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                         const nrtgpu_sort* sort, const nrtgpu_search_limits* limits, void* stream,
                         int32_t* out_docs, int64_t* out_sort_values, int32_t* out_counts,
                         int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout,
                         uint8_t* out_terminated_early);

/* Sort on several fields (a Sort of 1..8 SortFields, SortParser.parseSort :54-92; Sortable.java:34-45). Each field is
 *   NRTGPU_SORT_COLUMN  a numeric doc-value column (sortable-long domain), ascending unless reverse; a doc without a value
 *                       sorts as missing_value; on a MULTI-valued column `selector` picks the doc's smallest (MIN, the
 *                       default) or largest (MAX) value (SortedNumericSelector), ignored on a single-valued one;
 *   NRTGPU_SORT_DOCID   the doc id, ascending unless reverse; the fields after it cannot decide anything and are ignored;
 *   NRTGPU_SORT_SCORE   the BM25 score, higher first unless reverse (RelevanceComparator); FIRST position only;
 *   NRTGPU_SORT_KEYWORD a keyword column `column` (nrtgpu_index_add_keyword_columns) by its term in unsigned-byte order
 *                       (SortField STRING / SortedSetSortField), ascending unless reverse. On a SORTED_SET column the
 *                       selector picks one of the doc's n ascending ordinals: MIN ords[0], MAX ords[n-1], MIDDLE_MIN
 *                       ords[(n-1)/2], MIDDLE_MAX ords[n/2] (SortedSetSelector); it is ignored on a SORTED column.
 *                       missing_value 0 (STRING_FIRST): a doc without a value sorts before every term; 1 (STRING_LAST):
 *                       after every term. reverse reverses the whole comparison, the missing position included.
 *                       Its FieldDoc value (out_sort_values, after_values, nrtgpu_nested_sort.values, packed records) is
 *                       the term's code in the dictionary of the call: 2i + 2 for term i, 0 for no value (null). On a
 *                       single image that is the image's dictionary, on a searcher the reader-wide union. After values may
 *                       also hold 2i + 1 (i in 0..n): a term held by no dictionary, between term i - 1 and term i; any
 *                       other code is NRTGPU_ERR_INVALID. nrtgpu_index_keyword_seek / nrtgpu_searcher_keyword_seek turn a
 *                       term into its code; the *_keyword_term calls turn code c back (ordinal c / 2 - 1).
 * The implicit last tie-break is the doc id, ascending. An order (nrtgpu_sort_order) ranks every doc of the image under
 * one Sort once (an O(n log n) device sort on `stream`); it depends on the columns only, so it stays valid across
 * nrtgpu_index_set_live_docs and nrtgpu_index_update_stats: build one per (leaf, Sort) and reuse it for every request.
 * It holds 8 bytes per doc of device memory (nrtgpu_sort_order_device_bytes) and must be closed before its index.
 *   nrtgpu_sort_order_create: NRTGPU_ERR_INVALID for n_fields < 1, a bad kind or selector, a column out of range;
 *                             for a KEYWORD field also a keyword column out of range, a selector outside MIN..MIDDLE_MAX
 *                             and a missing_value other than 0 or 1 (MIDDLE_* on a COLUMN field is a bad selector);
 *                             NRTGPU_ERR_UNSUPPORTED for n_fields > 8 or a SCORE after the first position.
 *   nrtgpu_search_sorted (one field) keeps refusing the KEYWORD kind ("bad sort kind").
 *   nrtgpu_search_sorted_fields: as nrtgpu_search_sorted (exact totalHits, the same limits and refusals) with the order's
 *     Sort. out_sort_values [nq*top_k*n_fields] = FieldDoc.fields of every hit: a column's selected value or missing_value,
 *     the global doc id for DOCID, the score's float bits zero-extended for SCORE (Float.floatToIntBits).
 *     after_values [nq*n_fields] (same encoding) + nrtgpu_query.has_after / after_doc: a hit qualifies iff its field tuple
 *     sorts strictly after the after tuple, or ties with it and has a greater global doc id than after_doc
 *     (PagingFieldCollector); the values need not be held by any doc of this leaf.
 *     NRTGPU_ERR_INVALID: an order of another index, has_after without after_values, a KEYWORD after code outside
 *     0..2n + 1 (n: the column's terms). */
enum { NRTGPU_SORT_SCORE = 3, NRTGPU_SORT_KEYWORD = 5 };   /* (4 is taken by an internal kind) */
enum { NRTGPU_SELECT_MIN = 0, NRTGPU_SELECT_MAX = 1, NRTGPU_SELECT_MIDDLE_MIN = 2, NRTGPU_SELECT_MIDDLE_MAX = 3 };
typedef struct {
  int32_t kind;          /* NRTGPU_SORT_COLUMN, NRTGPU_SORT_DOCID, NRTGPU_SORT_SCORE or NRTGPU_SORT_KEYWORD */
  int32_t column;        /* NRTGPU_SORT_COLUMN: doc-value column id; NRTGPU_SORT_KEYWORD: keyword column id */
  int32_t reverse;
  int32_t selector;      /* NRTGPU_SELECT_MIN / _MAX (multi-valued columns); MIDDLE_MIN / _MAX: SORTED_SET keyword only */
  int64_t missing_value; /* NRTGPU_SORT_KEYWORD: 0 STRING_FIRST, 1 STRING_LAST */
} nrtgpu_sort_field;
typedef struct nrtgpu_sort_order nrtgpu_sort_order;
int nrtgpu_sort_order_create(nrtgpu_index* ix, const nrtgpu_sort_field* fields, int32_t n_fields, void* stream,
                             nrtgpu_sort_order** out);
int64_t nrtgpu_sort_order_device_bytes(const nrtgpu_sort_order* o);
int nrtgpu_sort_order_close(nrtgpu_sort_order* o);
int nrtgpu_search_sorted_fields(nrtgpu_index* ix, const nrtgpu_sort_order* order, const nrtgpu_clause* clauses,
                                int32_t n_clauses, const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                const int64_t* after_values, const nrtgpu_search_limits* limits, void* stream,
                                int32_t* out_docs, int64_t* out_sort_values, int32_t* out_counts,
                                int64_t* out_total_hits, uint8_t* out_relation, uint8_t* out_hit_timeout,
                                uint8_t* out_terminated_early);

/* Packed sorted result record: what TopFieldDocs.merge needs of one leaf or shard, in ONE device buffer (the sorted
 * counterpart of the score record of nrtgpu_packed_words). int32 words:
 *   docs [nq*top_k] (global ids) | counts [nq] | flags [nq] (bit 0: relation GTE, bit 1: terminated early, bit 2: hit
 *   timeout) | pad to 8 bytes | totalHits [nq] int64 | values [nq*top_k*n_fields] int64
 * values are out_sort_values of nrtgpu_search_sorted_fields (FieldDoc.fields of every hit); docs and values past counts[q]
 * are 0 in a merged record. nrtgpu_sorted_packed_words = record size in words (0 for nq or top_k <= 0, n_fields outside
 * 1..8); records must be 8-byte aligned.
 *   nrtgpu_search_sorted_fields_packed: nrtgpu_search_sorted_fields (the same refusals and results) with the results left
 *     in the caller-owned DEVICE record d_record; synchronises `stream`. With disallow_partial_results a timeout is
 *     NRTGPU_ERR_TIMEOUT, as on the host path.
 *   nrtgpu_merge_sorted_packed: TopFieldDocs.merge of n_lists records [n_lists][words] of the same Sort into d_out_record,
 *     on `stream` (asynchronous). fields = the Sort's nrtgpu_sort_field records; kind and reverse are read, and for a
 *     KEYWORD field missing_value. Hits compare field by field: COLUMN and DOCID by the value as a sortable long, ascending
 *     unless reverse; SCORE by the float of its bits, higher first unless reverse; KEYWORD by its code, code 0 first
 *     (missing_value 0) or last (1), the whole reversed with reverse. Keyword codes compare only when every record numbers
 *     them in one dictionary (a searcher maps its leaves' codes to the reader-wide union before it merges; records of
 *     different shards do not compare). The fields after the first DOCID are ignored; then the global doc id
 *     ascending. totalHits are summed and the flags ORed. NRTGPU_ERR_INVALID: n_lists < 1, n_fields outside 1..8, a bad
 *     kind, nq <= 0, top_k outside 1..1024, an unaligned record. */
int64_t nrtgpu_sorted_packed_words(int32_t nq, int32_t top_k, int32_t n_fields);
int nrtgpu_search_sorted_fields_packed(nrtgpu_index* ix, const nrtgpu_sort_order* order, const nrtgpu_clause* clauses,
                                       int32_t n_clauses, const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                       const int64_t* after_values, const nrtgpu_search_limits* limits, void* stream,
                                       int32_t* d_record);
int nrtgpu_merge_sorted_packed(nrtgpu_ctx* ctx, const nrtgpu_sort_field* fields, int32_t n_fields, int32_t n_lists, int32_t nq,
                               int32_t top_k, const int32_t* d_records, int32_t* d_out_record, void* stream);

/* Aggregating "additional collectors" over ALL docs matching each query (ScoreMode.COMPLETE: RelevanceCollector.java:55-62
 * forces totalHitsThreshold = MAX when additional collectors exist; fan-out SearchCollectorManager.java:192-198):
 *   NRTGPU_AGG_TERMS  counts per distinct value of a numeric doc-value column, the `size` buckets with the largest
 *                     (order_desc) or smallest counts, totalBuckets, totalOtherCounts
 *                     ({Int,Long,Float,Double}TermsCollectorManager + TermsCollectorManager.fillBucketResultByCount);
 *   NRTGPU_AGG_MIN / _MAX / _SUM   over the column's values as doubles (Min/Max/SumCollectorManager with the value
 *                     source doc['field'].value). MAX keeps `value > maxValue` started from -Double.MAX_VALUE, MIN
 *                     `value < minValue` from Double.MAX_VALUE: NaN never wins, nor does -inf for MAX or +inf for MIN
 *                     (a max over {-inf} is -Double.MAX_VALUE). A query with no match, or a batch with no work (every
 *                     query without clauses or with minimumNumberShouldMatch above its SHOULD count), gives
 *                     Double.MAX_VALUE / -Double.MAX_VALUE / 0.0, and a terms aggregation no buckets.
 * value_type says how the column's sortable long maps back to the number: 0 int / long, 1 float, 2 double.
 * Keyword terms (OrdinalTermsCollectorManager, TermsCollectorManager.java:154-170): a TERMS aggregation with value_type
 *   NRTGPU_AGG_VALUE_KEYWORD (3) counts keyword column `column` (nrtgpu_index_add_keyword_columns) per term. A doc of a
 *   SORTED_SET column counts once in the bucket of each of its terms (and is handed to the nested collectors once per
 *   term). bucket_keys are ordinals: the image's own, or on a searcher reader-wide ordinals into the byte-order union of
 *   the leaves' dictionaries (nrtgpu_index_keyword_term / nrtgpu_searcher_keyword_term give the bytes). Every other rule
 *   reads "value" as "term": size, order_desc, totalBuckets, totalOtherCounts, ties to the smaller term in byte order,
 *   the 2 GB nq x terms table (on a searcher with the union's term count), filters, nested collectors and the window
 *   engine, with no limit on a doc's terms. NRTGPU_ERR_INVALID: a keyword column out of range; MIN / MAX / SUM with value_type 3 keep "bad aggregation value_type" (a keyword has no
 *   number).
 * Docs without a value contribute nothing. Bucket ties at the cut are unordered in the reference (hash-map order); here
 * the smaller value wins. Min, max (up to the sign of a zero, which depends on collection order in the reference too)
 * and every count are exact. Sums are accumulated in a different order than the reference's single thread: for n finite
 * values the two differ by at most n * 2^-53 * sum|v| (an absolute bound: cancelling values lose the relative one), so
 * int / long sums with sum|v| < 2^53 are exact, and whether partial sums near Double.MAX_VALUE overflow depends on the
 * order in both; with a NaN, or both infinities, the sum is NaN, else with an infinity that infinity. */
enum { NRTGPU_AGG_TERMS = 1, NRTGPU_AGG_MIN = 2, NRTGPU_AGG_MAX = 3, NRTGPU_AGG_SUM = 4 };
enum { NRTGPU_AGG_VALUE_KEYWORD = 3 };   /* value_type of a terms aggregation over a keyword column */
typedef struct {
  int32_t kind, column, value_type;
  int32_t size;        /* terms: buckets returned (<= 2048) */
  int32_t order_desc;  /* terms: 1 = largest counts first (BucketOrder DESC by count, the default) */
  int32_t filter_agg;  /* terms / filter: 1 + the index of the FILTER aggregation this one is nested under; 0: top level
                          (nrtgpu_search_bool_aggs_filtered) */
} nrtgpu_aggregation;
typedef struct {       /* caller-allocated outputs of one aggregation (unused pointers may be NULL) */
  double* values;          /* [nq]        min / max / sum */
  int64_t* bucket_keys;    /* [nq*size]   terms: column values (sortable-long domain); keyword terms: ordinals */
  int32_t* bucket_counts;  /* [nq*size] */
  int32_t* n_buckets;      /* [nq]        buckets filled */
  int32_t* total_buckets;  /* [nq]        BucketResult.totalBuckets */
  int64_t* other_counts;   /* [nq]        BucketResult.totalOtherCounts */
} nrtgpu_aggregation_result;
/* nrtgpu_search_bool with additional collectors: hits as usual (exact totalHits), plus the aggregations */
int nrtgpu_search_bool_aggs(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                            const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                            const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                            void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                            int64_t* out_total_hits);

/* Nested collectors of a terms aggregation (search.proto Collector.nestedCollectors, CollectorCreator.java:73-126): each
 * is computed per bucket over exactly the docs its parent bucket counts (matching, live, with a value in the parent
 * column). A terms aggregation (aggs[parent]) carries up to 4:
 *   NRTGPU_AGG_MIN / _MAX / _SUM   over a single-valued column, with the rules of the top-level ones above (started from
 *                     +/-Double.MAX_VALUE, NaN never wins, the same sum bound); a bucket with no value in the column keeps
 *                     the unset value (Double.MAX_VALUE / -Double.MAX_VALUE / 0.0);
 *   NRTGPU_AGG_TOP_HITS  TopScoreDocCollectorManager(top_hits, null, Integer.MAX_VALUE) per bucket
 *                     (TopHitsCollectorManager.java:126-130): hits by score descending, then global doc ascending; positions
 *                     [start_hit, top_hits) are returned (:162), totalHits is the bucket's count (EQUAL_TO), and a score is
 *                     the float the top-level hit list gives that doc. Valid only as a nested kind.
 * orders_parent: at most one nested MIN / MAX / SUM of a parent orders its buckets instead of the count (BucketOrder by a
 * nested collector's name, TermsCollectorManager.fillBucketResultByNestedOrder :930-994), in the parent's order_desc
 * direction by Double.compare; ties, unordered in the reference's heap, go to the smaller bucket value; a bucket without
 * values takes part with the unset value. totalBuckets and totalOtherCounts keep their meaning.
 * Results are per returned bucket (the parent's `size` slots; entries past its n_buckets are 0):
 *   values [nq*size]   MIN / MAX / SUM of the bucket;
 *   TOP_HITS: hit_docs (global ids) / hit_scores [nq*size*(top_hits-start_hit)], hit_counts [nq*size] hits returned,
 *   hit_total [nq*size] the bucket's count.
 * Top hits are collected exactly in a second run of the batch's probe launch, after the buckets are chosen: the keys
 * (score, doc) of every collected doc of a returned bucket go into a buffer sized by the bucket's count, then one CTA per
 * bucket selects its best top_hits. The second run writes none of the request's hits, totalHits or aggregation tables.
 * When the buffers of the batch exceed 512 MB (2^26 keys) the second run goes over groups of queries.
 * nrtgpu_search_bool_aggs_nested: nrtgpu_search_bool_aggs (every refusal, the same hits and results) plus the nested
 * collectors; with n_nested == 0 it is nrtgpu_search_bool_aggs.
 *   NRTGPU_ERR_INVALID: a parent out of range or not a terms aggregation, a bad kind or value_type, a column out of range,
 *     start_hit outside [0, top_hits), two orders_parent on one parent (or on a TOP_HITS);
 *   NRTGPU_ERR_UNSUPPORTED: more than 4 nested collectors on a parent, a multi-valued nested column, top_hits > 1024,
 *     a batch x distinct values table of a nested metric over 2 GB, top-hit outputs over 2^24 entries per collector
 *     (nq * size * top_hits), a single query whose returned buckets hold more than 2^26 keys. */
enum { NRTGPU_AGG_TOP_HITS = 5 };
typedef struct {
  int32_t parent;         /* index into aggs[] of the terms (or filter) aggregation */
  int32_t kind;           /* NRTGPU_AGG_MIN / _MAX / _SUM / _TOP_HITS */
  int32_t column, value_type;   /* MIN / MAX / SUM */
  int32_t top_hits, start_hit;  /* TOP_HITS */
  int32_t orders_parent;  /* MIN / MAX / SUM: 1 = the parent's buckets are ordered by this value */
  int32_t reserved;
} nrtgpu_nested_aggregation;
typedef struct {          /* caller-allocated outputs of one nested collector (unused pointers may be NULL) */
  double* values;         /* [nq*size] */
  int32_t* hit_docs;      /* [nq*size*(top_hits-start_hit)] */
  float* hit_scores;      /* [nq*size*(top_hits-start_hit)] */
  int32_t* hit_counts;    /* [nq*size] */
  int64_t* hit_total;     /* [nq*size] */
} nrtgpu_nested_result;
int nrtgpu_search_bool_aggs_nested(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                                   const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                   const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                                   const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                                   const nrtgpu_nested_result* nested_results, void* stream, int32_t* out_docs,
                                   float* out_scores, int32_t* out_counts, int64_t* out_total_hits);

/* Filter collectors (search.proto Collector.filter, FilterCollectorManager.java): of the docs a query collects, those that
 * pass the filter are counted (docCount) and handed to the collectors nested under it.
 *   NRTGPU_AGG_FILTER  a top-level aggregation; its result is bucket_counts[nq], the query's docCount (the other result
 *                      pointers are unused). It needs a collector under it: a TERMS or FILTER aggregation whose filter_agg
 *                      names it, or a nested MIN / MAX / SUM / TOP_HITS whose parent it is; else NRTGPU_ERR_INVALID
 *                      'Filter collector "aggs[i]" must have nested collectors'.
 *   filter_agg         (nrtgpu_aggregation) 1 + the index of an EARLIER FILTER aggregation: a TERMS aggregation then counts,
 *                      and a FILTER aggregation passes, only the docs that pass that filter (a filter under a filter: both
 *                      must pass). Only TERMS and FILTER aggregations may set it; a MIN / MAX / SUM under a filter is a
 *                      nested collector of it. A terms aggregation under a filter keeps every terms rule above.
 *   nested collectors  parent may name a FILTER aggregation: MIN / MAX / SUM / TOP_HITS over the docs that pass, at most 4,
 *                      orders_parent refused. Results use the terms layout with size 1: values [nq], hit_docs / hit_scores
 *                      [nq*(top_hits-start_hit)], hit_counts [nq], hit_total [nq] = docCount.
 * The filter of a FILTER aggregation is agg_filters[i] (an array parallel to aggs, read for FILTER aggregations only):
 *   NRTGPU_AGG_FILTER_QUERY      filter_queries[query], a flat BooleanQuery in the clause format of nrtgpu_search_bool over
 *                      filter_clauses (QueryFilter: only matching counts, boosts and scores are ignored). The kNN filters'
 *                      rules apply: has_after is NRTGPU_ERR_INVALID, more than 16 clauses or 8 term clauses
 *                      NRTGPU_ERR_UNSUPPORTED, an empty clause range or MUST_NOT clauses only match nothing.
 *   NRTGPU_AGG_FILTER_VALUE_SET  values[n_values] in the sortable-long domain of `column` (SetQueryFilter over a
 *                      TermInSetQuery): a doc passes when one of its values (a single-valued or multi-valued column) is in
 *                      the set, by bit equality in that domain, so -0.0 != 0.0 and NaN == NaN as in Java's boxed equals.
 *                      Any order, duplicates allowed; n_values == 0 passes nothing. A set of another term type than the
 *                      field's never matches in the reference: the caller passes an empty set.
 *   NRTGPU_AGG_FILTER_KEYWORD_SET  values[n_values] are keyword codes (nrtgpu_index_keyword_seek; reader-wide codes on a
 *                      searcher) of keyword column `column` (SetQueryFilter over the TEXTTERMS of an atom field): a doc passes
 *                      when the code of one of its terms is in the set (String equals). An odd code is a term the dictionary
 *                      does not hold and matches nothing. NRTGPU_ERR_INVALID: a keyword column out of range, a code outside
 *                      [1, 2n + 1].
 * Every query of the batch takes the same filters. Deleted docs never pass.
 * nrtgpu_search_bool_aggs_filtered: nrtgpu_search_bool_aggs_nested (every refusal, the same hits and results) plus filter
 * collectors; nrtgpu_search_bool_aggs and _aggs_nested are this call without filter records.
 *   NRTGPU_ERR_INVALID: a FILTER aggregation without agg_filters, a bad record kind, a query or column out of range,
 *     n_values < 0 or values NULL with n_values > 0, a filter_agg that is not an earlier FILTER aggregation or set on a MIN /
 *     MAX / SUM, orders_parent under a FILTER parent, a FILTER aggregation nothing is nested under.
 *   The 8-aggregation cap counts the FILTER aggregations. Query trees and wide batches stay NRTGPU_ERR_UNSUPPORTED. A refused
 *   call writes no output. */
enum { NRTGPU_AGG_FILTER = 6 };
enum { NRTGPU_AGG_FILTER_QUERY = 1, NRTGPU_AGG_FILTER_VALUE_SET = 2, NRTGPU_AGG_FILTER_KEYWORD_SET = 4 };   /* (3 stays a bad filter kind) */
typedef struct {
  int32_t kind;           /* NRTGPU_AGG_FILTER_QUERY / _VALUE_SET / _KEYWORD_SET */
  int32_t query;          /* QUERY: index into filter_queries */
  int32_t column;         /* VALUE_SET: numeric column; KEYWORD_SET: keyword column */
  int32_t n_values;       /* VALUE_SET, KEYWORD_SET */
  const int64_t* values;  /* VALUE_SET: [n_values] sortable longs; KEYWORD_SET: [n_values] keyword codes */
} nrtgpu_agg_filter;
int nrtgpu_search_bool_aggs_filtered(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                                     const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                     const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                                     const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                                     const nrtgpu_nested_result* nested_results, const nrtgpu_agg_filter* agg_filters,
                                     const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses,
                                     const nrtgpu_query* filter_queries, int32_t n_filter_queries, void* stream,
                                     int32_t* out_docs, float* out_scores, int32_t* out_counts, int64_t* out_total_hits);

/* Sorted top hits (TopHitsCollector with a querySort: TopHitsCollectorManager.java:126-130 uses
 * TopFieldCollectorManager(sort, top_hits, null, Integer.MAX_VALUE) instead of the score collector). nested_sorts is an
 * array parallel to `nested` (NULL: every top hits by score); entry j, read for a TOP_HITS record only:
 *   orders   NULL: by score, exactly as nrtgpu_search_bool_aggs_filtered. Else the Sort's nrtgpu_sort_order: orders[0] on
 *            the single image; one per leaf, in leaf order, for a searcher (as nrtgpu_searcher_search_sorted_fields takes
 *            them). The bucket's docs are ordered by the Sort with the rules of nrtgpu_search_sorted_fields: a column
 *            ascending unless reverse, missing_value for a doc without a value, the MIN / MAX selector on a multi-valued
 *            column; DOCID the global doc id; a leading SCORE the float the top-level hit list gives that doc. Ties go to
 *            the smaller global doc. Positions [start_hit, top_hits) are returned, hit_total is the bucket's count.
 *            hit_scores are NaN (the reduce sets Hit.score = Double.NaN); a leading SCORE's value is in `values`.
 *   values   NULL, or [nq*size*(top_hits-start_hit)*n_fields] (size 1 under a FILTER parent): FieldDoc.fields of every
 *            returned hit, in the encoding of out_sort_values of nrtgpu_search_sorted_fields; 0 past hit_counts.
 * A top-level TopHitsCollector ("the page by relevance, plus the 5 newest matches") is the nested top hits of a FILTER
 * aggregation whose filter query is match-all: every doc the query collects passes, so hit_total is the query's totalHits.
 * On a searcher each leaf selects its own top_hits of a bucket by its order, and the leaves' lists are merged as
 * TopFieldDocs.merge does (nrtgpu_merge_sorted_packed); the lists of one pass-2 group of queries take
 * (n_leaves + 1) * nq_group * size * (top_hits * (1 + 2 * n_fields) + 4) * 4 bytes per sorted collector, and the groups
 * are cut so that this stays under 512 MB unless one query needs more by itself.
 * nrtgpu_search_bool_aggs_filtered is this call without nested_sorts.
 *   NRTGPU_ERR_INVALID, beside every refusal of nrtgpu_search_bool_aggs_filtered: orders on a record that is not TOP_HITS,
 *     a NULL order, an order made on another index (or, for a searcher, another leaf), leaf orders of different Sorts.
 *     orders_parent on a TOP_HITS stays 'top hits cannot order the buckets'. The 8-field limit and the SCORE-first rule are
 *     nrtgpu_sort_order_create's. A refused call writes no output. */
typedef struct {
  const nrtgpu_sort_order* const* orders;   /* NULL: by score; else [1] (single image) or [n_leaves] (searcher) */
  int64_t* values;                          /* [nq*size*(top_hits-start_hit)*n_fields] or NULL */
} nrtgpu_nested_sort;
int nrtgpu_search_bool_aggs_sorted_hits(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                                        const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                        const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                                        const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                                        const nrtgpu_nested_result* nested_results, const nrtgpu_nested_sort* nested_sorts,
                                        const nrtgpu_agg_filter* agg_filters, const nrtgpu_clause* filter_clauses,
                                        int32_t n_filter_clauses, const nrtgpu_query* filter_queries, int32_t n_filter_queries,
                                        void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                                        int64_t* out_total_hits);
/* nrtgpu_search_tree_aggs: nrtgpu_search_bool_aggs_sorted_hits for the queries of nrtgpu_search_tree_phrases ("deep dish
 * pizza" as a match_phrase or a multi_match, by category, plus the 3 best per category). The batch takes the tree and phrase
 * arguments of nrtgpu_search_tree_phrases (n_nodes / n_phrases may be 0; nodes / phrases may then be NULL) and every
 * collector argument of nrtgpu_search_bool_aggs_sorted_hits, with its meaning and result layout. A batch holding a nested
 * query or a phrase, or a flat batch of more than 4 term clauses or top_k > 512, runs on the window engine
 * (bool_window_kernel), which hands every matching doc and its score to the collectors, and runs again for the nested top
 * hits; any other flat batch runs on the probe kernel exactly as nrtgpu_search_bool_aggs_sorted_hits runs it. The page and
 * totalHits are those of nrtgpu_search_tree_phrases at totalHitsThreshold = INT32_MAX (totalHits exact).
 *   Every refusal of nrtgpu_search_tree_phrases and of nrtgpu_search_bool_aggs_sorted_hits applies with its code and message,
 *   but for "aggregations over a query tree" and "aggregations: more than 4 term clauses or top_k > 512", which this call
 *   accepts. A refused call writes no output. */
int nrtgpu_search_tree_aggs(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes, int32_t n_nodes,
                            const nrtgpu_phrase* phrases, int32_t n_phrases, const nrtgpu_phrase_term* phrase_terms,
                            int32_t n_phrase_terms, const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                            const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                            const nrtgpu_nested_aggregation* nested, int32_t n_nested, const nrtgpu_nested_result* nested_results,
                            const nrtgpu_nested_sort* nested_sorts, const nrtgpu_agg_filter* agg_filters,
                            const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses, const nrtgpu_query* filter_queries,
                            int32_t n_filter_queries, void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                            int64_t* out_total_hits);

/* QueryRescorer second pass (QueryRescore.java:39-57 -> Lucene QueryRescorer.rescore): query q of the batch evaluated on
 * ITS OWN hit list docs[q][0..counts[q]) (global doc ids): out_matches / out_scores [nq*n_hits]. */
int nrtgpu_score_docs(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                      const nrtgpu_query* queries, int32_t nq, int32_t n_hits, const int32_t* docs,
                      const int32_t* counts /*[nq] or NULL*/, void* stream, uint8_t* out_matches, float* out_scores);
/* The whole rescore on the device, Lucene QueryRescorer.rescore(searcher, hits, topN = windowSize) as QueryRescore.java:52-57
 * calls it: second pass over EVERY first-pass hit + QueryRescore.combine (double math -> float) + re-sort
 * (score desc, doc asc), in place; out_counts[q] = min(counts[q], window) hits are kept.
 * docs / scores [nq*n_hits] HOST buffers (in/out), n_hits <= 4096. */
int nrtgpu_rescore_query(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                         const nrtgpu_query* queries, int32_t nq, int32_t n_hits, const int32_t* counts,
                         int32_t window, double query_weight, double rescore_weight, void* stream,
                         int32_t* docs, float* scores, int32_t* out_counts /*[nq] or NULL*/);
/* The same pair for rescore queries that are query trees or hold phrases (a QueryRescorer whose rescore query is a
 * match_phrase, a multi_match or a bool of those). They take the tree and phrase arguments of nrtgpu_search_tree_phrases and
 * keep the semantics of nrtgpu_score_docs / nrtgpu_rescore_query: global doc ids, counts may be NULL in score_docs, a doc
 * outside the leaf, a deleted doc and an entry past counts[q] get match 0 and score 0. A matching doc's score is the float
 * the window engine gives the same doc for the same tree (the node rules of nrtgpu_search_tree, the phrase weight and freq
 * rules of nrtgpu_search_tree_phrases). Every refusal of nrtgpu_search_tree_phrases applies, and every argument check of the
 * flat pair. With n_nodes == 0 and n_phrases == 0 they are nrtgpu_score_docs / nrtgpu_rescore_query; a batch holding a
 * nested query or a phrase is evaluated as a tree batch, its flat queries included. */
int nrtgpu_score_docs_tree(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                           int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                           const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                           int32_t nq, int32_t n_hits, const int32_t* docs, const int32_t* counts /*[nq] or NULL*/,
                           void* stream, uint8_t* out_matches, float* out_scores);
int nrtgpu_rescore_query_tree(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                              int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                              const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                              int32_t nq, int32_t n_hits, const int32_t* counts, int32_t window, double query_weight,
                              double rescore_weight, void* stream, int32_t* docs, float* scores,
                              int32_t* out_counts /*[nq] or NULL*/);

/* Fetch phase on doc-value columns (SearchHandler.java:397-522, FillDocsTask.fetchFromDocVales / LoadedDocValues): the
 * values of n_cols columns for n hits (global doc ids): out_values / out_has [n_cols*n]. */
int nrtgpu_fetch_columns(nrtgpu_index* ix, const int32_t* col_ids, int32_t n_cols, const int32_t* docs, int32_t n,
                         void* stream, int64_t* out_values, uint8_t* out_has);

/* Split form: compile+upload once, launch many times with everything resident in HBM (query trees:
 * nrtgpu_batch_prepare_tree). A prepared batch holds the weights and score bounds of the statistics it was compiled with:
 * it stays valid across nrtgpu_index_set_live_docs; after nrtgpu_index_update_stats prepare it again. */
int nrtgpu_batch_prepare(nrtgpu_index* ix, const nrtgpu_clause* clauses, int32_t n_clauses,
                         const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                         int32_t total_hits_threshold, int32_t flags, nrtgpu_batch** out);
int nrtgpu_batch_run(nrtgpu_batch* b, void* stream);   /* asynchronous: kernels only */
int nrtgpu_batch_fetch(nrtgpu_batch* b, void* stream, int32_t* out_docs, float* out_scores,
                       int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation);
int nrtgpu_batch_set_limits(nrtgpu_batch* b, const nrtgpu_search_limits* limits);   /* NULL clears; applies to later runs */
int nrtgpu_batch_fetch_ex(nrtgpu_batch* b, void* stream, int32_t* out_docs, float* out_scores,
                          int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation,
                          uint8_t* out_hit_timeout, uint8_t* out_terminated_early);
/* device pointers of the last run's results: uint64 keys are not exposed; these are the final arrays */
int nrtgpu_batch_device_results(nrtgpu_batch* b, int32_t** d_docs, float** d_scores, int32_t** d_counts);
/* redirect the final (docs, scores, counts) of subsequent runs into caller-owned DEVICE buffers
 * ([nq*top_k], [nq*top_k], [nq]); NULLs restore the internal buffers */
int nrtgpu_batch_bind_output(nrtgpu_batch* b, int32_t* d_docs, float* d_scores, int32_t* d_counts);
/* Packed per-shard result record: the ONE buffer a multi-GPU step all-gathers (docs, scores, counts, relation /
 * terminated flags and totalHits of every query). int32 words:
 *   docs [nq*top_k] | scores [nq*top_k] (float bits) | counts [nq] | flags [nq] (bit 0: relation GTE, bit 1: terminated
 *   early) | pad to 8 bytes | totalHits [nq] int64.      nrtgpu_packed_words = record size in words.
 * nrtgpu_batch_bind_packed redirects the results of subsequent runs into a caller-owned DEVICE record (NULL restores
 * the internal buffers); nrtgpu_merge_topk_packed is TopDocs.merge over n_lists gathered records (totalHits summed,
 * relation GTE if any shard's is: LazyQueueTopScoreDocCollectorManager.java:137-144) into one record, on the device.
 * Every score-ranked page of top_k slots (this record, the bound or internal outputs of a batch, nrtgpu_merge_topk_device,
 * nrtgpu_searcher_search_bool, nrtgpu_blend_rrf / _scores) holds its count hits first; the slots past the count hold
 * doc 0 and score 0.0, whatever an earlier request left in the buffer (a sorted page keeps NaN scores there). */
int64_t nrtgpu_packed_words(int32_t nq, int32_t top_k);
int nrtgpu_batch_bind_packed(nrtgpu_batch* b, int32_t* d_record);
int nrtgpu_merge_topk_packed(nrtgpu_ctx* ctx, int32_t n_lists, int32_t nq, int32_t top_k, const int32_t* d_records,
                             int32_t* d_out_record, void* stream);

/* stats of the compiled batch: algorithmic postings (sum of df over all term clauses), kernel launches per run */
int nrtgpu_batch_stats(const nrtgpu_batch* b, int64_t* alg_postings, int32_t* launches_per_run,
                       int64_t* work_items);
/* mean duration (ms) of stage `stage` over the runs since nrtgpu_batch_reset_timing (at most the last
 * 64; CUDA events recorded on each run's stream, which must have been synchronised).
 * stage 0 = posting traversal kernel, 1 = slice merge kernel. */
int nrtgpu_batch_stage_ms(nrtgpu_batch* b, int32_t stage, float* ms);
int nrtgpu_batch_reset_timing(nrtgpu_batch* b);
int nrtgpu_batch_free(nrtgpu_batch* b);

/* Exact kNN (ExactVectorQuery / KnnFloatVectorQuery with exact semantics): HOST buffers. Deleted docs (live_docs of the
 * shard) are never hits, as through IndexSearcher's acceptDocs; `filter` is ANDed on top. Exact BY CONSTRUCTION: the
 * tensor-core candidate stage is followed by an fp64 re-score and a rank-safety certificate (every vector outside the
 * candidate list is proven, with the bf16 error bound 2^-7 |q||d|, to score below the k-th exact score); queries the
 * certificate rejects are re-run by exact evaluation of every vector (nrtgpu_knn_last_uncertified counts them).
 * NRTGPU_ERR_INVALID: nq <= 0, k outside 1..1024, an index without vectors, or a boost that is not a BoostQuery boost:
 * every boosts[q] must be finite and >= 0 (negative, -0, NaN and infinite boosts are refused, as Lucene's BoostQuery does;
 * with a negative boost the final order would be the reverse of the candidate order and the certificate would accept the
 * worst vectors). Boost 0 is legal: every score is 0 and the page holds the first k docs. The same rule holds for
 * nrtgpu_search_knn_filtered; nrtgpu_search_knn_timed takes no boosts and refuses nq <= 0. */
int nrtgpu_search_knn(nrtgpu_index* ix, const float* queries, int32_t nq, int32_t k,
                      const float* boosts /*[nq] or NULL*/, const uint8_t* filter /*[n_docs] 0/1 or NULL*/,
                      void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts);

/* same search, plus the device time (ms, CUDA events on `stream`) of its three stages:
 * stage_ms[0] candidate GEMM (wgmma bf16 when dims % 8 == 0), [1] per-query select, [2] exact fp64 re-score */
int nrtgpu_search_knn_timed(nrtgpu_index* ix, const float* queries, int32_t nq, int32_t k, void* stream,
                            int32_t* out_docs, float* out_scores, int32_t* out_counts, float* stage_ms);

/* number of queries of the most recent kNN call on this index that took the exact fallback */
int32_t nrtgpu_knn_last_uncertified(const nrtgpu_index* ix);

/* Exact kNN in which every query has its own filter query (KnnQuery.filter, reference KnnUtils.java:135-155). The filters
 * are flat BooleanQuerys in the same clause format as nrtgpu_search_bool, and they are evaluated on the device.
 *   filters[n_filters]: clause ranges into filter_clauses. Only matching counts: boosts and scores are ignored.
 *   filter_of[nq]: index into filters, or -1 for no filter. Queries that share a filter pass the same index, and
 *   each filter is evaluated once per call.
 * Deleted docs never match. Results are as for nrtgpu_search_knn: the exact top-k among the docs that match the query's
 * filter, so counts[q] < k when fewer match. Matching follows the boolean path: an empty clause range matches nothing, as an
 * empty BooleanQuery does; so does a query of MUST_NOT clauses only.
 * NRTGPU_ERR_INVALID: has_after on a filter, a filter_of entry or clause id out of range, an index without vectors, k outside
 * 1..1024, nq <= 0, a boost that is negative, -0, NaN or infinite. NRTGPU_ERR_UNSUPPORTED: a filter shape outside the boolean path (more than 16 clauses or 8 term clauses); the
 * byte filter of nrtgpu_search_knn still serves it.
 * A query whose filter matches at most 1/320 of the vectors is scored exactly over those docs only; the others go through
 * the candidate GEMM with the filter applied. The first path needs one vector per doc in doc order (ascending vec_docs, as
 * Lucene assigns vector ordinals); on a shard whose vec_docs is not strictly ascending every query takes the second.
 * Device scratch is bounded: the filter bitmaps of one call (one row of n_docs / 8 bytes per distinct filter) are capped at
 * 128 MB, and a call with more distinct filters runs in groups of queries whose rows fit; the term bitmaps they are built
 * from are capped at another 128 MB. nrtgpu_knn_last_uncertified counts this call's exact fallbacks. */
int nrtgpu_search_knn_filtered(nrtgpu_index* ix, const float* queries, int32_t nq, int32_t k, const float* boosts,
                               const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses,
                               const nrtgpu_query* filters, int32_t n_filters, const int32_t* filter_of,
                               void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts);

/* of the most recent nrtgpu_search_knn_filtered call on this index: queries scored over their filter's docs only (the rest
 * took the candidate GEMM), and the device time of the filter evaluation in ms (either pointer may be NULL) */
int nrtgpu_knn_filter_stats(const nrtgpu_index* ix, int32_t* out_gather_queries, float* out_filter_ms);

/* TopDocs.merge over `n_lists` per-shard lists resident on the DEVICE (the receive buffer of the NCCL
 * all-gather): docs/scores [n_lists][nq][top_k], counts [n_lists][nq]; outputs on the device. */
int nrtgpu_merge_topk_device(nrtgpu_ctx* ctx, int32_t n_lists, int32_t nq, int32_t top_k,
                             const int32_t* d_docs, const float* d_scores, const int32_t* d_counts,
                             int32_t* d_out_docs, float* d_out_scores, int32_t* d_out_counts, void* stream);

/* Weighted RRF blend of R retrievers' lists for nq queries (HOST buffers):
 * docs [R][nq][top_in], counts [R][nq], boosts [R]; out [nq][top_out]. */
int nrtgpu_blend_rrf(nrtgpu_ctx* ctx, int32_t n_retrievers, int32_t nq, int32_t top_in,
                     const int32_t* docs, const int32_t* counts, const float* boosts,
                     int32_t rank_constant, int32_t top_out, int32_t* out_docs, float* out_scores,
                     int32_t* out_counts, int32_t* out_total);

/* Score-order blend (WeightedScoreOrderBlenderOperation.java:50-73 with WeightedScoreDoc.java:57-77): every hit contributes
 * score * boost of its retriever; a doc found by several retrievers combines them, in retriever declaration order and in
 * float, by MAX (default), SUM or AVG (running average). scores [R][nq][top_in]; other arguments as nrtgpu_blend_rrf. */
enum { NRTGPU_BLEND_MAX = 1, NRTGPU_BLEND_SUM = 2, NRTGPU_BLEND_AVG = 3 };
int nrtgpu_blend_scores(nrtgpu_ctx* ctx, int32_t score_mode, int32_t n_retrievers, int32_t nq, int32_t top_in,
                        const int32_t* docs, const float* scores, const int32_t* counts, const float* boosts,
                        int32_t top_out, int32_t* out_docs, float* out_scores, int32_t* out_counts, int32_t* out_total);

/* QueryRescore.combine + re-sort for nq hit lists (HOST buffers, in place): [nq][n_hits]. */
int nrtgpu_rescore_combine(nrtgpu_ctx* ctx, int32_t nq, int32_t n_hits, const int32_t* counts,
                           int32_t* docs, float* scores, const uint8_t* second_matches,
                           const float* second_scores, double query_weight, double rescore_weight);

/* ---- NRT refresh without rebuilding images (ShardSearcherFactory.newSearcher(reader, previous), ShardState.java:506-526).
 * A shard is searched through ONE image per Lucene leaf (segment); the adaptor numbers (field, term) once per shard, so
 * clause ids mean the same term in every leaf. A new reader version keeps the images of the leaves it shares with the
 * previous one and builds images only for the NEW leaves (nrtgpu_index_build with the leaf's docBase); what changes for
 * the old leaves is
 *   - their liveDocs (deletes):               nrtgpu_index_set_live_docs   (NULL = no deletes)
 *   - the index-wide statistics BM25 uses:     nrtgpu_index_update_stats    (docFreq per term, docCount and
 *     sumTotalTermFreq per field; refreshes the idf inputs, the length caches and the index-time impact bounds).
 * Both wait for searches in flight on the image. nrtgpu_searcher = the leaves of one reader version: every leaf runs the
 * batch, the per-leaf pages are merged on the device (TopDocs.merge), totalHits summed, relation GTE if any leaf's is.
 * The searcher does not own the leaves. */
int nrtgpu_index_set_live_docs(nrtgpu_index* ix, const uint8_t* live_docs /*[n_docs] 0/1 or NULL*/);
int nrtgpu_index_update_stats(nrtgpu_index* ix, const int64_t* term_df /*[n_terms] or NULL = unchanged*/,
                              const int64_t* field_doc_count /*[n_fields]*/, const int64_t* field_sum_ttf /*[n_fields]*/);
typedef struct nrtgpu_searcher nrtgpu_searcher;
int nrtgpu_searcher_create(nrtgpu_ctx* ctx, nrtgpu_index* const* leaves, int32_t n_leaves, nrtgpu_searcher** out);
int nrtgpu_searcher_search_bool(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses,
                                const nrtgpu_query* queries, int32_t nq, int32_t top_k,
                                int32_t total_hits_threshold, int32_t flags, const nrtgpu_search_limits* limits,
                                void* stream, int32_t* out_docs, float* out_scores, int32_t* out_counts,
                                int64_t* out_total_hits, uint8_t* out_relation);
int nrtgpu_searcher_close(nrtgpu_searcher* s);
/* The other top-k searches over the leaves: every leaf runs the request into a device record (the leaves' searches are
 * sequential), the records are merged on the device, the merged page is copied to the host outputs (any may be NULL).
 * Every refusal of the single-image entry point applies: the first failing leaf's code is returned and no output is
 * written. Limits are handed to every leaf unchanged, as by nrtgpu_searcher_search_bool; a leaf's hit_timeout /
 * terminated_early / relation GTE make the merged query's.
 *   nrtgpu_searcher_search_sorted_fields: nrtgpu_search_sorted_fields over the leaves (TopFieldDocs.merge,
 *     nrtgpu_merge_sorted_packed). orders[n_orders]: one nrtgpu_sort_order per leaf, in leaf order, all of the same Sort (the
 *     same kinds and directions, and for a column or keyword field the same column, selector and missing value).
 *     after_values / after_doc are reader-wide and go to every leaf unchanged, except a KEYWORD field's code, which each
 *     leaf receives in its own dictionary (nrtgpu_searcher_keyword_seek). A one-field Sort is a one-field order here.
 *     NRTGPU_ERR_INVALID: n_orders != the number of leaves, an order made on another index than its leaf, orders of
 *     different Sorts.
 *   nrtgpu_searcher_search_tree_phrases: nrtgpu_search_tree_phrases over the leaves (n_nodes / n_phrases may be 0);
 *     TopDocs.merge of the leaves' pages by nrtgpu_merge_topk_packed.
 *   nrtgpu_searcher_search_knn / _filtered: the single-image kNN searches over the leaves (per-leaf exact top-k, then
 *     TopDocs.merge by score desc, doc asc). filter: one byte per global doc id (leaf l reads filter[doc_base ..
 *     doc_base + n_docs)). A leaf without vectors contributes no hits; NRTGPU_ERR_INVALID when no leaf has vectors. */
int nrtgpu_searcher_search_sorted_fields(nrtgpu_searcher* s, const nrtgpu_sort_order* const* orders, int32_t n_orders,
                                         const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_query* queries, int32_t nq,
                                         int32_t top_k, int32_t flags, const int64_t* after_values,
                                         const nrtgpu_search_limits* limits, void* stream, int32_t* out_docs,
                                         int64_t* out_sort_values, int32_t* out_counts, int64_t* out_total_hits,
                                         uint8_t* out_relation, uint8_t* out_hit_timeout, uint8_t* out_terminated_early);
int nrtgpu_searcher_search_tree_phrases(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                                        int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                                        const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                                        int32_t nq, int32_t top_k, int32_t total_hits_threshold, int32_t flags,
                                        const nrtgpu_search_limits* limits, void* stream, int32_t* out_docs, float* out_scores,
                                        int32_t* out_counts, int64_t* out_total_hits, uint8_t* out_relation,
                                        uint8_t* out_hit_timeout, uint8_t* out_terminated_early);
int nrtgpu_searcher_search_knn(nrtgpu_searcher* s, const float* queries, int32_t nq, int32_t k, const float* boosts /*[nq] or NULL*/,
                               const uint8_t* filter /*one byte per global doc or NULL*/, void* stream, int32_t* out_docs,
                               float* out_scores, int32_t* out_counts);
int nrtgpu_searcher_search_knn_filtered(nrtgpu_searcher* s, const float* queries, int32_t nq, int32_t k, const float* boosts,
                                        const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses, const nrtgpu_query* filters,
                                        int32_t n_filters, const int32_t* filter_of, void* stream, int32_t* out_docs,
                                        float* out_scores, int32_t* out_counts);
/* nrtgpu_searcher_search_bool_aggs_nested: nrtgpu_search_bool_aggs_nested over the leaves (n_nested may be 0). Terms buckets
 * are counted by value across the leaves, as TermsCollectorManager.reduce merges its per-slice maps: each leaf numbers a
 * column's values in its own dictionary, so the first aggregation on a column builds the searcher's reader-wide dictionary
 * of it (the union of the leaves' distinct values, and per leaf its doc codes renumbered to it: 4 B per doc, except in a
 * leaf whose dictionary is the union or that holds no value), kept until nrtgpu_searcher_close. Every leaf counts into one
 * set of tables of nq x U buckets (U: the union's size), and buckets, totalBuckets, otherCounts and the nested values are
 * selected once from them. Nested top hits are chosen per reader-wide bucket over every leaf's hits, ties by global doc; the
 * scores are the leaves' own, the shard's when the leaves carry the index-wide statistics. The page is TopDocs.merge of the
 * leaves' pages (nrtgpu_merge_topk_packed); totalHits is exact and summed over the leaves.
 *   Every refusal of nrtgpu_search_bool_aggs_nested applies with the same code and message, on every leaf: query trees and
 *   wide batches are NRTGPU_ERR_UNSUPPORTED, so is a column multi-valued in any leaf; a column index some leaf lacks is
 *   NRTGPU_ERR_INVALID. The 2 GB limits of the count and nested-word tables apply at the reader-wide U: a batch whose leaves
 *   each fit but whose union does not is refused before any batch is built or table allocated. On a refusal no output is
 *   written. NULL searcher: NRTGPU_ERR_INVALID.
 * Keyword terms over the leaves: the reader-wide dictionary of a keyword column is the byte-order union of the leaves' term
 * dictionaries, built on the host by its first aggregation (or nrtgpu_searcher_keyword_term) and kept until close; each
 * leaf's ordinals are mapped to it (its codes renumbered: 4 B per doc for SORTED, per value for SORTED_SET, except in a
 * leaf whose dictionary is the union). bucket_keys are ordinals of the union. A keyword column index some leaf lacks is
 * NRTGPU_ERR_INVALID. */
/* The bytes of reader-wide term `ord` of keyword column `column` (as nrtgpu_index_keyword_term); builds the column's
 * reader-wide dictionary if no call has yet, on the default stream. *n_terms (may be NULL) receives the union's size.
 * NRTGPU_ERR_INVALID: a column some leaf lacks, an ordinal out of range (ord -1 only asks for n_terms), len NULL. */
int nrtgpu_searcher_keyword_term(nrtgpu_searcher* s, int32_t column, int32_t ord, uint8_t* out, int32_t cap, int32_t* len,
                                 int32_t* n_terms);
/* nrtgpu_index_keyword_seek in the reader-wide dictionary of keyword column `column` (built as by
 * nrtgpu_searcher_keyword_term if no call has yet): the after values of nrtgpu_searcher_search_sorted_fields and the
 * values it returns for a KEYWORD field are codes of that dictionary. Each leaf is searched with the code its own
 * dictionary gives the same term, and its hits' codes are mapped to the union on the device before the merge; sorted top
 * hits over the leaves likewise. NRTGPU_ERR_INVALID: a column some leaf lacks, and the refusals of the image call. */
int nrtgpu_searcher_keyword_seek(nrtgpu_searcher* s, int32_t column, const uint8_t* bytes, int32_t len, int64_t* code);
/* nrtgpu_index_keyword_range in the reader-wide dictionary of keyword column `column`: the code range of an
 * NRTGPU_KEYWORD_RANGE clause on a searcher. Keyword clauses (in queries, filter queries and kNN filter queries) and keyword
 * value sets of a searcher carry reader-wide codes; each leaf receives them mapped to its own dictionary. NRTGPU_ERR_INVALID:
 * a column some leaf lacks, and the refusals of the image call. */
int nrtgpu_searcher_keyword_range(nrtgpu_searcher* s, int32_t column, const uint8_t* lower, int32_t lower_len,
                                  const uint8_t* upper, int32_t upper_len, int32_t flags, int64_t* lo, int64_t* hi);
int nrtgpu_searcher_search_bool_aggs_nested(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses,
                                            const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                            const nrtgpu_aggregation* aggs, int32_t n_aggs, const nrtgpu_aggregation_result* results,
                                            const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                                            const nrtgpu_nested_result* nested_results, void* stream, int32_t* out_docs,
                                            float* out_scores, int32_t* out_counts, int64_t* out_total_hits);
/* nrtgpu_searcher_search_bool_aggs_filtered: nrtgpu_search_bool_aggs_filtered over the leaves, with the rules above. Each leaf
 * evaluates the filters on its own image; every leaf counts into the one set of tables, so docCount and the values nested
 * under a filter are reader-wide, a terms aggregation under a filter uses the reader-wide dictionary, and top hits under a
 * filter are chosen over every leaf, ties by global doc. nrtgpu_searcher_search_bool_aggs_nested is this call without
 * filter records. */
int nrtgpu_searcher_search_bool_aggs_filtered(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses,
                                              const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                              const nrtgpu_aggregation* aggs, int32_t n_aggs,
                                              const nrtgpu_aggregation_result* results, const nrtgpu_nested_aggregation* nested,
                                              int32_t n_nested, const nrtgpu_nested_result* nested_results,
                                              const nrtgpu_agg_filter* agg_filters, const nrtgpu_clause* filter_clauses,
                                              int32_t n_filter_clauses, const nrtgpu_query* filter_queries,
                                              int32_t n_filter_queries, void* stream, int32_t* out_docs, float* out_scores,
                                              int32_t* out_counts, int64_t* out_total_hits);
/* nrtgpu_searcher_search_bool_aggs_sorted_hits: nrtgpu_search_bool_aggs_sorted_hits over the leaves (one order per leaf in
 * nested_sorts[j].orders); sorted top hits are selected per leaf and merged as TopFieldDocs.merge does, ties by global doc;
 * top hits by score are chosen over every leaf at once as before. nrtgpu_searcher_search_bool_aggs_filtered is this call
 * without nested_sorts. */
int nrtgpu_searcher_search_bool_aggs_sorted_hits(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses,
                                                 const nrtgpu_query* queries, int32_t nq, int32_t top_k, int32_t flags,
                                                 const nrtgpu_aggregation* aggs, int32_t n_aggs,
                                                 const nrtgpu_aggregation_result* results,
                                                 const nrtgpu_nested_aggregation* nested, int32_t n_nested,
                                                 const nrtgpu_nested_result* nested_results, const nrtgpu_nested_sort* nested_sorts,
                                                 const nrtgpu_agg_filter* agg_filters, const nrtgpu_clause* filter_clauses,
                                                 int32_t n_filter_clauses, const nrtgpu_query* filter_queries,
                                                 int32_t n_filter_queries, void* stream, int32_t* out_docs, float* out_scores,
                                                 int32_t* out_counts, int64_t* out_total_hits);
/* nrtgpu_searcher_search_tree_aggs: nrtgpu_search_tree_aggs over the leaves, with the rules of
 * nrtgpu_searcher_search_bool_aggs_sorted_hits (reader-wide tables and dictionaries, one order per leaf, sorted top hits
 * merged as TopFieldDocs.merge does, the page by TopDocs.merge). Every leaf runs the batch on the same engine. */
int nrtgpu_searcher_search_tree_aggs(nrtgpu_searcher* s, const nrtgpu_clause* clauses, int32_t n_clauses, const nrtgpu_node* nodes,
                                     int32_t n_nodes, const nrtgpu_phrase* phrases, int32_t n_phrases,
                                     const nrtgpu_phrase_term* phrase_terms, int32_t n_phrase_terms, const nrtgpu_query* queries,
                                     int32_t nq, int32_t top_k, int32_t flags, const nrtgpu_aggregation* aggs, int32_t n_aggs,
                                     const nrtgpu_aggregation_result* results, const nrtgpu_nested_aggregation* nested,
                                     int32_t n_nested, const nrtgpu_nested_result* nested_results,
                                     const nrtgpu_nested_sort* nested_sorts, const nrtgpu_agg_filter* agg_filters,
                                     const nrtgpu_clause* filter_clauses, int32_t n_filter_clauses,
                                     const nrtgpu_query* filter_queries, int32_t n_filter_queries, void* stream, int32_t* out_docs,
                                     float* out_scores, int32_t* out_counts, int64_t* out_total_hits);

/* Request micro-batcher: the reference's search API is ONE query per RPC (clientlib/src/main/proto/yelp/nrtsearch/
 * luceneserver.proto:164), each on its own SERVER-pool thread (GrpcServerExecutorSupplier.java:68-75). Handler threads call
 * nrtgpu_batcher_submit (blocking) with one flat BooleanQuery; a worker thread owned by the batcher groups the waiting requests
 * that share (top_k, totalHitsThreshold) into one nrtgpu_search_bool call as soon as max_batch of them wait or the oldest has
 * waited max_wait_us, and scatters the results. A request that fails compilation is re-run alone, so it cannot fail its
 * neighbours. nrtgpu_diagnostics carries what SearchResponse.Diagnostics reports per search (SearchHandler.java:261,280,321):
 * time queued, time of the batched search, and the size of the batch the request rode in. */
typedef struct nrtgpu_batcher nrtgpu_batcher;
typedef struct { double queue_ms; double search_ms; int32_t batch_size; int32_t reserved; } nrtgpu_diagnostics;
int nrtgpu_batcher_create(nrtgpu_index* ix, int32_t max_batch, int32_t max_wait_us, nrtgpu_batcher** out);
int nrtgpu_batcher_submit(nrtgpu_batcher* b, const nrtgpu_clause* clauses, int32_t n_clauses, int32_t min_should_match,
                          int32_t top_k, int32_t total_hits_threshold, int32_t* out_docs, float* out_scores,
                          int32_t* out_count, int64_t* out_total_hits, uint8_t* out_relation,
                          nrtgpu_diagnostics* diag /* or NULL */);
int nrtgpu_batcher_stats(nrtgpu_batcher* b, int64_t* n_batches, int64_t* n_requests);
int nrtgpu_batcher_close(nrtgpu_batcher* b);   /* drains the queue, joins the worker */

#ifdef __cplusplus
}
#endif
#endif
