/*
 * nrtgpu_jni.c -- thin JNI shim over include/nrtgpu.h (pure marshalling; every decision is behind the C ABI).
 * NOT compiled in this repository's image (no JDK / jni.h here); build on the server host with
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude jni/nrtgpu_jni.c \
 *       -Lnrtsearch_b200 -lnrtgpu -o libnrtgpu_jni.so
 * Java side: jni/java/com/yelp/nrtsearch/server/gpu/NrtGpu.java. Buffers are direct ByteBuffers (caller allocated).
 */
#include <jni.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "nrtgpu.h"

#define ADDR(env, buf) ((buf) ? (*(env))->GetDirectBufferAddress((env), (buf)) : NULL)

static jint fail(JNIEnv* env, int rc) {
  if (rc == NRTGPU_OK) return 0;
  const char* cls = rc == NRTGPU_ERR_INVALID ? "java/lang/IllegalArgumentException"
                  : rc == NRTGPU_ERR_UNSUPPORTED ? "java/lang/UnsupportedOperationException"
                  : rc == NRTGPU_ERR_TIMEOUT ? "com/yelp/nrtsearch/server/search/collectors/CollectionTimeoutException"
                  : "java/lang/RuntimeException";   /* -> Status.INTERNAL in SearchHandler.handle (:136-145) */
  (*env)->ThrowNew(env, (*env)->FindClass(env, cls), nrtgpu_last_error());
  return rc;
}

JNIEXPORT jlong JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_init(JNIEnv* env, jclass c, jint device) {
  nrtgpu_ctx* ctx = NULL;
  if (fail(env, nrtgpu_init(device, &ctx))) return 0;
  return (jlong)(intptr_t)ctx;
}
JNIEXPORT void JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_shutdown(JNIEnv* env, jclass c, jlong ctx) {
  nrtgpu_shutdown((nrtgpu_ctx*)(intptr_t)ctx);
}
/* desc: a direct ByteBuffer laid out as nrtgpu_shard_desc (pointers = addresses of other direct buffers) */
JNIEXPORT jlong JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_indexBuild(JNIEnv* env, jclass c, jlong ctx, jobject desc) {
  nrtgpu_index* ix = NULL;
  if (fail(env, nrtgpu_index_build((nrtgpu_ctx*)(intptr_t)ctx, (const nrtgpu_shard_desc*)ADDR(env, desc), &ix))) return 0;
  return (jlong)(intptr_t)ix;
}
JNIEXPORT void JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_indexClose(JNIEnv* env, jclass c, jlong ix) {
  nrtgpu_index_close((nrtgpu_index*)(intptr_t)ix);
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchBool(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK,
    jint totalHitsThreshold, jint flags, jobject outDocs, jobject outScores, jobject outCounts, jobject outTotalHits,
    jobject outRelation) {
  return fail(env, nrtgpu_search_bool((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                      (const nrtgpu_query*)ADDR(env, queries), nq, topK, totalHitsThreshold, flags, NULL,
                                      (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores), (int32_t*)ADDR(env, outCounts),
                                      (int64_t*)ADDR(env, outTotalHits), (uint8_t*)ADDR(env, outRelation)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchKnn(
    JNIEnv* env, jclass c, jlong ix, jobject queries, jint nq, jint k, jobject boosts, jobject filter, jobject outDocs,
    jobject outScores, jobject outCounts) {
  return fail(env, nrtgpu_search_knn((nrtgpu_index*)(intptr_t)ix, (const float*)ADDR(env, queries), nq, k,
                                     (const float*)ADDR(env, boosts), (const uint8_t*)ADDR(env, filter), NULL,
                                     (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores), (int32_t*)ADDR(env, outCounts)));
}
/* filterClauses / filters: direct buffers laid out as nrtgpu_clause[] / nrtgpu_query[]; filterOf: int32 per query (-1 = none) */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchKnnFiltered(
    JNIEnv* env, jclass c, jlong ix, jobject queries, jint nq, jint k, jobject boosts, jobject filterClauses,
    jint nFilterClauses, jobject filters, jint nFilters, jobject filterOf, jobject outDocs, jobject outScores, jobject outCounts) {
  return fail(env, nrtgpu_search_knn_filtered((nrtgpu_index*)(intptr_t)ix, (const float*)ADDR(env, queries), nq, k,
                                              (const float*)ADDR(env, boosts), (const nrtgpu_clause*)ADDR(env, filterClauses),
                                              nFilterClauses, (const nrtgpu_query*)ADDR(env, filters), nFilters,
                                              (const int32_t*)ADDR(env, filterOf), NULL, (int32_t*)ADDR(env, outDocs),
                                              (float*)ADDR(env, outScores), (int32_t*)ADDR(env, outCounts)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_blendRrf(
    JNIEnv* env, jclass c, jlong ctx, jint nRetrievers, jint nq, jint topIn, jobject docs, jobject counts, jobject boosts,
    jint rankConstant, jint topOut, jobject outDocs, jobject outScores, jobject outCounts, jobject outTotal) {
  return fail(env, nrtgpu_blend_rrf((nrtgpu_ctx*)(intptr_t)ctx, nRetrievers, nq, topIn, (const int32_t*)ADDR(env, docs),
                                    (const int32_t*)ADDR(env, counts), (const float*)ADDR(env, boosts), rankConstant, topOut,
                                    (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores), (int32_t*)ADDR(env, outCounts),
                                    (int32_t*)ADDR(env, outTotal)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_rescoreCombine(
    JNIEnv* env, jclass c, jlong ctx, jint nq, jint nHits, jobject counts, jobject docs, jobject scores, jobject secondMatches,
    jobject secondScores, jdouble queryWeight, jdouble rescoreWeight) {
  return fail(env, nrtgpu_rescore_combine((nrtgpu_ctx*)(intptr_t)ctx, nq, nHits, (const int32_t*)ADDR(env, counts),
                                          (int32_t*)ADDR(env, docs), (float*)ADDR(env, scores),
                                          (const uint8_t*)ADDR(env, secondMatches), (const float*)ADDR(env, secondScores),
                                          queryWeight, rescoreWeight));
}

/* limits: a direct ByteBuffer laid out as nrtgpu_search_limits (or null); sort: nrtgpu_sort */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchBoolEx(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK,
    jint totalHitsThreshold, jint flags, jobject limits, jobject outDocs, jobject outScores, jobject outCounts,
    jobject outTotalHits, jobject outRelation, jobject outHitTimeout, jobject outTerminatedEarly) {
  return fail(env, nrtgpu_search_bool_ex((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                         (const nrtgpu_query*)ADDR(env, queries), nq, topK, totalHitsThreshold, flags,
                                         (const nrtgpu_search_limits*)ADDR(env, limits), NULL, (int32_t*)ADDR(env, outDocs),
                                         (float*)ADDR(env, outScores), (int32_t*)ADDR(env, outCounts),
                                         (int64_t*)ADDR(env, outTotalHits), (uint8_t*)ADDR(env, outRelation),
                                         (uint8_t*)ADDR(env, outHitTimeout), (uint8_t*)ADDR(env, outTerminatedEarly)));
}
/* nodes: a direct ByteBuffer laid out as nrtgpu_node[] (28 bytes each: kind, clause_begin, clause_end, min_should_match,
 * tie_breaker, boost, min_score; null with nNodes 0: the search of searchBoolEx) */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchTree(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject nodes, jint nNodes, jobject queries, jint nq,
    jint topK, jint totalHitsThreshold, jint flags, jobject limits, jobject outDocs, jobject outScores, jobject outCounts,
    jobject outTotalHits, jobject outRelation, jobject outHitTimeout, jobject outTerminatedEarly) {
  return fail(env, nrtgpu_search_tree((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                      (const nrtgpu_node*)ADDR(env, nodes), nNodes, (const nrtgpu_query*)ADDR(env, queries), nq,
                                      topK, totalHitsThreshold, flags, (const nrtgpu_search_limits*)ADDR(env, limits), NULL,
                                      (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores), (int32_t*)ADDR(env, outCounts),
                                      (int64_t*)ADDR(env, outTotalHits), (uint8_t*)ADDR(env, outRelation),
                                      (uint8_t*)ADDR(env, outHitTimeout), (uint8_t*)ADDR(env, outTerminatedEarly)));
}
/* positions: a direct ByteBuffer of int32 positions, posting after posting (PostingsEnum.nextPosition()) */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_addPositions(JNIEnv* env, jclass c, jlong ix, jobject positions,
                                                                               jlong nPositions) {
  return fail(env, nrtgpu_index_add_positions((nrtgpu_index*)(intptr_t)ix, (const int32_t*)ADDR(env, positions), nPositions));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_addParents(JNIEnv* env, jclass c, jlong ix, jint rootTerm) {
  return fail(env, nrtgpu_index_add_parents((nrtgpu_index*)(intptr_t)ix, rootTerm));
}
/* keyword columns (SortedDocValues / SortedSetDocValues of the leaf), column k from element k of each array: termBytes,
 * termOffsets (int64[nTerms + 1]), ords (int32) and docOffsets (int64[maxDoc + 1], SORTED_SET; null for SORTED) are direct
 * ByteBuffers */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_addKeywordColumns(JNIEnv* env, jclass c, jlong ix, jintArray nTerms,
                                                                                   jintArray multiValued, jobjectArray termBytes,
                                                                                   jobjectArray termOffsets, jobjectArray ords,
                                                                                   jobjectArray docOffsets) {
  const jsize n = nTerms ? (*env)->GetArrayLength(env, nTerms) : 0;
  if (n > 0 && (!multiValued || !termBytes || !termOffsets || !ords || !docOffsets || (*env)->GetArrayLength(env, multiValued) != n ||
                (*env)->GetArrayLength(env, termBytes) != n || (*env)->GetArrayLength(env, termOffsets) != n ||
                (*env)->GetArrayLength(env, ords) != n || (*env)->GetArrayLength(env, docOffsets) != n)) {
    (*env)->ThrowNew(env, (*env)->FindClass(env, "java/lang/IllegalArgumentException"),
                     "addKeywordColumns: the six arrays must have one element per column");
    return NRTGPU_ERR_INVALID;
  }
  nrtgpu_keyword_column* cols = (nrtgpu_keyword_column*)calloc(n > 0 ? (size_t)n : 1, sizeof(nrtgpu_keyword_column));
  if (!cols) return fail(env, NRTGPU_ERR_OOM);
  jint* nt = n ? (*env)->GetIntArrayElements(env, nTerms, NULL) : NULL;
  jint* mv = n ? (*env)->GetIntArrayElements(env, multiValued, NULL) : NULL;
  for (jsize k = 0; k < n; ++k) {
    cols[k].n_terms = nt[k]; cols[k].multi_valued = mv[k];
    jobject tb = (*env)->GetObjectArrayElement(env, termBytes, k), to = (*env)->GetObjectArrayElement(env, termOffsets, k);
    jobject od = (*env)->GetObjectArrayElement(env, ords, k), dof = (*env)->GetObjectArrayElement(env, docOffsets, k);
    cols[k].term_bytes = (const uint8_t*)ADDR(env, tb);
    cols[k].term_offsets = (const int64_t*)ADDR(env, to);
    cols[k].ords = (const int32_t*)ADDR(env, od);
    cols[k].doc_offsets = (const int64_t*)ADDR(env, dof);
    /* the direct buffers stay reachable from the caller's arrays: their addresses outlive these local references */
    if (tb) (*env)->DeleteLocalRef(env, tb);
    if (to) (*env)->DeleteLocalRef(env, to);
    if (od) (*env)->DeleteLocalRef(env, od);
    if (dof) (*env)->DeleteLocalRef(env, dof);
  }
  if (n) { (*env)->ReleaseIntArrayElements(env, nTerms, nt, JNI_ABORT); (*env)->ReleaseIntArrayElements(env, multiValued, mv, JNI_ABORT); }
  const int rc = nrtgpu_index_add_keyword_columns((nrtgpu_index*)(intptr_t)ix, cols, n);
  free(cols);
  return fail(env, rc);
}
/* the bytes of a keyword term into out (at most cap of them); returns the term's length */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_keywordTerm(JNIEnv* env, jclass c, jlong ix, jint column, jint ord,
                                                                             jobject out, jint cap) {
  int32_t len = 0;
  if (fail(env, nrtgpu_index_keyword_term((const nrtgpu_index*)(intptr_t)ix, column, ord, (uint8_t*)ADDR(env, out), cap, &len))) return -1;
  return len;
}
/* a reader-wide keyword term of a searcher (ord -1: the term count of the union is returned) */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searcherKeywordTerm(JNIEnv* env, jclass c, jlong s, jint column,
                                                                                     jint ord, jobject out, jint cap) {
  int32_t len = 0, n_terms = 0;
  if (fail(env, nrtgpu_searcher_keyword_term((nrtgpu_searcher*)(intptr_t)s, column, ord, (uint8_t*)ADDR(env, out), cap, &len, &n_terms)))
    return -1;
  return ord == -1 ? n_terms : len;
}
/* the sort code of a keyword term (term: a direct ByteBuffer of len bytes) in an image's dictionary: a LastHitInfo string
 * as the after value of an NRTGPU_SORT_KEYWORD field; -1 after a refusal (the exception is pending) */
JNIEXPORT jlong JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_keywordSeek(JNIEnv* env, jclass c, jlong ix, jint column, jobject term,
                                                                              jint len) {
  int64_t code = 0;
  if (fail(env, nrtgpu_index_keyword_seek((const nrtgpu_index*)(intptr_t)ix, column, (const uint8_t*)ADDR(env, term), len, &code))) return -1;
  return code;
}
/* keywordSeek in a searcher's reader-wide dictionary */
JNIEXPORT jlong JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searcherKeywordSeek(JNIEnv* env, jclass c, jlong s, jint column,
                                                                                      jobject term, jint len) {
  int64_t code = 0;
  if (fail(env, nrtgpu_searcher_keyword_seek((nrtgpu_searcher*)(intptr_t)s, column, (const uint8_t*)ADDR(env, term), len, &code))) return -1;
  return code;
}
/* the code range [lo, hi] of a keyword range clause (NRTGPU_KEYWORD_RANGE) from term bounds (direct ByteBuffers; flags
 * NRTGPU_KEYWORD_*: NO_LOWER 1, NO_UPPER 2, LOWER_EXCLUSIVE 4, UPPER_EXCLUSIVE 8, PREFIX 16) into out[0..1] (a direct
 * ByteBuffer of two longs), in an image's dictionary (searcher == 0) or a searcher's reader-wide one; 0 or the refusal's code */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_keywordRange(JNIEnv* env, jclass c, jlong ix, jlong s, jint column,
                                                                              jobject lower, jint lowerLen, jobject upper,
                                                                              jint upperLen, jint flags, jobject out) {
  int64_t* o = (int64_t*)ADDR(env, out);
  const uint8_t* lo = (const uint8_t*)ADDR(env, lower);
  const uint8_t* hi = (const uint8_t*)ADDR(env, upper);
  return s ? fail(env, nrtgpu_searcher_keyword_range((nrtgpu_searcher*)(intptr_t)s, column, lo, lowerLen, hi, upperLen, flags, o, o + 1))
           : fail(env, nrtgpu_index_keyword_range((const nrtgpu_index*)(intptr_t)ix, column, lo, lowerLen, hi, upperLen, flags, o, o + 1));
}
/* phrases / phraseTerms: direct ByteBuffers laid out as nrtgpu_phrase[] / nrtgpu_phrase_term[] (nPhrases 0: searchTree),
 * for clauses of kind NRTGPU_PHRASE and NRTGPU_MULTI_PHRASE */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchTreePhrases(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject nodes, jint nNodes, jobject phrases, jint nPhrases,
    jobject phraseTerms, jint nPhraseTerms, jobject queries, jint nq, jint topK, jint totalHitsThreshold, jint flags,
    jobject limits, jobject outDocs, jobject outScores, jobject outCounts, jobject outTotalHits, jobject outRelation,
    jobject outHitTimeout, jobject outTerminatedEarly) {
  return fail(env, nrtgpu_search_tree_phrases((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                              (const nrtgpu_node*)ADDR(env, nodes), nNodes,
                                              (const nrtgpu_phrase*)ADDR(env, phrases), nPhrases,
                                              (const nrtgpu_phrase_term*)ADDR(env, phraseTerms), nPhraseTerms,
                                              (const nrtgpu_query*)ADDR(env, queries), nq, topK, totalHitsThreshold, flags,
                                              (const nrtgpu_search_limits*)ADDR(env, limits), NULL, (int32_t*)ADDR(env, outDocs),
                                              (float*)ADDR(env, outScores), (int32_t*)ADDR(env, outCounts),
                                              (int64_t*)ADDR(env, outTotalHits), (uint8_t*)ADDR(env, outRelation),
                                              (uint8_t*)ADDR(env, outHitTimeout), (uint8_t*)ADDR(env, outTerminatedEarly)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchSorted(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK, jint flags,
    jobject sort, jobject limits, jobject outDocs, jobject outSortValues, jobject outCounts, jobject outTotalHits,
    jobject outRelation, jobject outHitTimeout, jobject outTerminatedEarly) {
  return fail(env, nrtgpu_search_sorted((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                        (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                        (const nrtgpu_sort*)ADDR(env, sort), (const nrtgpu_search_limits*)ADDR(env, limits), NULL,
                                        (int32_t*)ADDR(env, outDocs), (int64_t*)ADDR(env, outSortValues),
                                        (int32_t*)ADDR(env, outCounts), (int64_t*)ADDR(env, outTotalHits),
                                        (uint8_t*)ADDR(env, outRelation), (uint8_t*)ADDR(env, outHitTimeout),
                                        (uint8_t*)ADDR(env, outTerminatedEarly)));
}
/* fields: a direct ByteBuffer of nFields nrtgpu_sort_field; the order handle goes to outOrder (a direct ByteBuffer of 8 bytes) */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_sortOrderCreate(
    JNIEnv* env, jclass c, jlong ix, jobject fields, jint nFields, jobject outOrder) {
  return fail(env, nrtgpu_sort_order_create((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_sort_field*)ADDR(env, fields), nFields, NULL,
                                            (nrtgpu_sort_order**)ADDR(env, outOrder)));
}
JNIEXPORT jlong JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_sortOrderDeviceBytes(JNIEnv* env, jclass c, jlong order) {
  return (jlong)nrtgpu_sort_order_device_bytes((const nrtgpu_sort_order*)(intptr_t)order);
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_sortOrderClose(JNIEnv* env, jclass c, jlong order) {
  return fail(env, nrtgpu_sort_order_close((nrtgpu_sort_order*)(intptr_t)order));
}
/* afterValues: nq * nFields int64 (FieldDoc.fields) or null */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchSortedFields(
    JNIEnv* env, jclass c, jlong ix, jlong order, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK, jint flags,
    jobject afterValues, jobject limits, jobject outDocs, jobject outSortValues, jobject outCounts, jobject outTotalHits,
    jobject outRelation, jobject outHitTimeout, jobject outTerminatedEarly) {
  return fail(env, nrtgpu_search_sorted_fields((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_sort_order*)(intptr_t)order,
                                               (const nrtgpu_clause*)ADDR(env, clauses), nClauses, (const nrtgpu_query*)ADDR(env, queries),
                                               nq, topK, flags, (const int64_t*)ADDR(env, afterValues),
                                               (const nrtgpu_search_limits*)ADDR(env, limits), NULL, (int32_t*)ADDR(env, outDocs),
                                               (int64_t*)ADDR(env, outSortValues), (int32_t*)ADDR(env, outCounts),
                                               (int64_t*)ADDR(env, outTotalHits), (uint8_t*)ADDR(env, outRelation),
                                               (uint8_t*)ADDR(env, outHitTimeout), (uint8_t*)ADDR(env, outTerminatedEarly)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_scoreDocs(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject queries, jint nq, jint nHits, jobject docs,
    jobject counts, jobject outMatches, jobject outScores) {
  return fail(env, nrtgpu_score_docs((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                     (const nrtgpu_query*)ADDR(env, queries), nq, nHits, (const int32_t*)ADDR(env, docs),
                                     (const int32_t*)ADDR(env, counts), NULL, (uint8_t*)ADDR(env, outMatches),
                                     (float*)ADDR(env, outScores)));
}
/* the second pass of a tree / phrase rescore query: the tree and phrase buffers as searchTreePhrases */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_scoreDocsTree(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject nodes, jint nNodes, jobject phrases, jint nPhrases,
    jobject phraseTerms, jint nPhraseTerms, jobject queries, jint nq, jint nHits, jobject docs, jobject counts,
    jobject outMatches, jobject outScores) {
  return fail(env, nrtgpu_score_docs_tree((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                          (const nrtgpu_node*)ADDR(env, nodes), nNodes, (const nrtgpu_phrase*)ADDR(env, phrases),
                                          nPhrases, (const nrtgpu_phrase_term*)ADDR(env, phraseTerms), nPhraseTerms,
                                          (const nrtgpu_query*)ADDR(env, queries), nq, nHits, (const int32_t*)ADDR(env, docs),
                                          (const int32_t*)ADDR(env, counts), NULL, (uint8_t*)ADDR(env, outMatches),
                                          (float*)ADDR(env, outScores)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_rescoreQueryTree(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject nodes, jint nNodes, jobject phrases, jint nPhrases,
    jobject phraseTerms, jint nPhraseTerms, jobject queries, jint nq, jint nHits, jobject counts, jint window,
    jdouble queryWeight, jdouble rescoreWeight, jobject docs, jobject scores, jobject outCounts) {
  return fail(env, nrtgpu_rescore_query_tree((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                             (const nrtgpu_node*)ADDR(env, nodes), nNodes, (const nrtgpu_phrase*)ADDR(env, phrases),
                                             nPhrases, (const nrtgpu_phrase_term*)ADDR(env, phraseTerms), nPhraseTerms,
                                             (const nrtgpu_query*)ADDR(env, queries), nq, nHits, (const int32_t*)ADDR(env, counts),
                                             window, queryWeight, rescoreWeight, NULL, (int32_t*)ADDR(env, docs),
                                             (float*)ADDR(env, scores), (int32_t*)ADDR(env, outCounts)));
}
/* additional collectors with nested collectors. aggs / nested: direct ByteBuffers of nrtgpu_aggregation[nAggs] /
 * nrtgpu_nested_aggregation[nNested]; aggOut: 6 direct buffers (or null) per aggregation in nrtgpu_aggregation_result field
 * order, nestedOut: 5 per nested collector in nrtgpu_nested_result field order. agg_results unpacks aggOut / nestedOut into
 * the result records (freed by the caller, also when it fails). */
static int agg_results(JNIEnv* env, jobjectArray aggOut, jint nAggs, jobjectArray nestedOut, jint nNested,
                       nrtgpu_aggregation_result** out_ar, nrtgpu_nested_result** out_nr) {
  nrtgpu_aggregation_result* ar = *out_ar = (nrtgpu_aggregation_result*)calloc(nAggs > 0 ? (size_t)nAggs : 1, sizeof(*ar));
  nrtgpu_nested_result* nr = *out_nr = (nrtgpu_nested_result*)calloc(nNested > 0 ? (size_t)nNested : 1, sizeof(*nr));
  if (!ar || !nr) return NRTGPU_ERR_OOM;
  for (jint i = 0; i < nAggs; ++i) {
    void* p[6];
    for (int f = 0; f < 6; ++f) p[f] = ADDR(env, (*env)->GetObjectArrayElement(env, aggOut, 6 * i + f));
    ar[i].values = (double*)p[0]; ar[i].bucket_keys = (int64_t*)p[1]; ar[i].bucket_counts = (int32_t*)p[2];
    ar[i].n_buckets = (int32_t*)p[3]; ar[i].total_buckets = (int32_t*)p[4]; ar[i].other_counts = (int64_t*)p[5];
  }
  for (jint i = 0; i < nNested; ++i) {
    void* p[5];
    for (int f = 0; f < 5; ++f) p[f] = ADDR(env, (*env)->GetObjectArrayElement(env, nestedOut, 5 * i + f));
    nr[i].values = (double*)p[0]; nr[i].hit_docs = (int32_t*)p[1]; nr[i].hit_scores = (float*)p[2];
    nr[i].hit_counts = (int32_t*)p[3]; nr[i].hit_total = (int64_t*)p[4];
  }
  return NRTGPU_OK;
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchBoolAggsNested(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK, jint flags,
    jobject aggs, jint nAggs, jobjectArray aggOut, jobject nested, jint nNested, jobjectArray nestedOut, jobject outDocs,
    jobject outScores, jobject outCounts, jobject outTotalHits) {
  nrtgpu_aggregation_result* ar = NULL;
  nrtgpu_nested_result* nr = NULL;
  int rc = agg_results(env, aggOut, nAggs, nestedOut, nNested, &ar, &nr);
  if (!rc)
    rc = nrtgpu_search_bool_aggs_nested((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                        (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                        (const nrtgpu_aggregation*)ADDR(env, aggs), nAggs, ar,
                                        (const nrtgpu_nested_aggregation*)ADDR(env, nested), nNested, nr, NULL,
                                        (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores),
                                        (int32_t*)ADDR(env, outCounts), (int64_t*)ADDR(env, outTotalHits));
  free(ar);
  free(nr);
  return fail(env, rc);
}
/* filter collectors: aggFilters = a direct ByteBuffer of nrtgpu_agg_filter[nAggs] (the values fields are ignored), filterValues
 * one direct buffer of int64 (or null) per aggregation, the value set of a VALUE_SET filter. agg_filter_records copies the
 * records with their values pointers set (freed by the caller, also when it fails); a null aggFilters gives NULL. */
static int agg_filter_records(JNIEnv* env, jobject aggFilters, jobjectArray filterValues, jint nAggs, nrtgpu_agg_filter** out) {
  *out = NULL;
  const void* src = ADDR(env, aggFilters);
  if (!src || nAggs <= 0) return NRTGPU_OK;
  nrtgpu_agg_filter* f = *out = (nrtgpu_agg_filter*)calloc((size_t)nAggs, sizeof(*f));
  if (!f) return NRTGPU_ERR_OOM;
  memcpy(f, src, (size_t)nAggs * sizeof(*f));
  for (jint i = 0; i < nAggs; ++i)
    f[i].values = filterValues ? (const int64_t*)ADDR(env, (*env)->GetObjectArrayElement(env, filterValues, i)) : NULL;
  return NRTGPU_OK;
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchBoolAggsFiltered(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK, jint flags,
    jobject aggs, jint nAggs, jobjectArray aggOut, jobject nested, jint nNested, jobjectArray nestedOut, jobject aggFilters,
    jobjectArray filterValues, jobject filterClauses, jint nFilterClauses, jobject filterQueries, jint nFilterQueries,
    jobject outDocs, jobject outScores, jobject outCounts, jobject outTotalHits) {
  nrtgpu_aggregation_result* ar = NULL;
  nrtgpu_nested_result* nr = NULL;
  nrtgpu_agg_filter* af = NULL;
  int rc = agg_results(env, aggOut, nAggs, nestedOut, nNested, &ar, &nr);
  if (!rc) rc = agg_filter_records(env, aggFilters, filterValues, nAggs, &af);
  if (!rc)
    rc = nrtgpu_search_bool_aggs_filtered((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                          (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                          (const nrtgpu_aggregation*)ADDR(env, aggs), nAggs, ar,
                                          (const nrtgpu_nested_aggregation*)ADDR(env, nested), nNested, nr, af,
                                          (const nrtgpu_clause*)ADDR(env, filterClauses), nFilterClauses,
                                          (const nrtgpu_query*)ADDR(env, filterQueries), nFilterQueries, NULL,
                                          (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores),
                                          (int32_t*)ADDR(env, outCounts), (int64_t*)ADDR(env, outTotalHits));
  free(ar);
  free(nr);
  free(af);
  return fail(env, rc);
}
/* the nrtgpu_nested_sort records of nested collector j: sortOrders[j] a long[] of sort-order handles (one per image; null:
 * by score), sortValues[j] a direct buffer for the FieldDoc values (or null). *orders holds the handle arrays (freed by
 * the caller with free_nested_sorts). */
static int nested_sort_records(JNIEnv* env, jobjectArray sortOrders, jobjectArray sortValues, jint nNested, nrtgpu_nested_sort** out,
                               const nrtgpu_sort_order*** orders) {
  *out = NULL; *orders = NULL;
  if (!sortOrders || nNested <= 0) return NRTGPU_OK;
  nrtgpu_nested_sort* s = *out = (nrtgpu_nested_sort*)calloc((size_t)nNested, sizeof(*s));
  const nrtgpu_sort_order** o = *orders = (const nrtgpu_sort_order**)calloc((size_t)nNested * 64, sizeof(*o));
  if (!s || !o) return NRTGPU_ERR_OOM;
  for (jint j = 0; j < nNested; ++j) {
    jlongArray h = (jlongArray)(*env)->GetObjectArrayElement(env, sortOrders, j);
    if (!h) continue;
    const jsize n = (*env)->GetArrayLength(env, h);
    if (n > 64) return NRTGPU_ERR_INVALID;
    jlong* v = (*env)->GetLongArrayElements(env, h, NULL);
    for (jsize l = 0; l < n; ++l) o[(size_t)j * 64 + l] = (const nrtgpu_sort_order*)(intptr_t)v[l];
    (*env)->ReleaseLongArrayElements(env, h, v, JNI_ABORT);
    s[j].orders = o + (size_t)j * 64;
    s[j].values = sortValues ? (int64_t*)ADDR(env, (*env)->GetObjectArrayElement(env, sortValues, j)) : NULL;
  }
  return NRTGPU_OK;
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchBoolAggsSortedHits(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK, jint flags,
    jobject aggs, jint nAggs, jobjectArray aggOut, jobject nested, jint nNested, jobjectArray nestedOut, jobjectArray sortOrders,
    jobjectArray sortValues, jobject aggFilters, jobjectArray filterValues, jobject filterClauses, jint nFilterClauses,
    jobject filterQueries, jint nFilterQueries, jobject outDocs, jobject outScores, jobject outCounts, jobject outTotalHits) {
  nrtgpu_aggregation_result* ar = NULL;
  nrtgpu_nested_result* nr = NULL;
  nrtgpu_agg_filter* af = NULL;
  nrtgpu_nested_sort* ns = NULL;
  const nrtgpu_sort_order** so = NULL;
  int rc = agg_results(env, aggOut, nAggs, nestedOut, nNested, &ar, &nr);
  if (!rc) rc = agg_filter_records(env, aggFilters, filterValues, nAggs, &af);
  if (!rc) rc = nested_sort_records(env, sortOrders, sortValues, nNested, &ns, &so);
  if (!rc)
    rc = nrtgpu_search_bool_aggs_sorted_hits((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                             (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                             (const nrtgpu_aggregation*)ADDR(env, aggs), nAggs, ar,
                                             (const nrtgpu_nested_aggregation*)ADDR(env, nested), nNested, nr, ns, af,
                                             (const nrtgpu_clause*)ADDR(env, filterClauses), nFilterClauses,
                                             (const nrtgpu_query*)ADDR(env, filterQueries), nFilterQueries, NULL,
                                             (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores),
                                             (int32_t*)ADDR(env, outCounts), (int64_t*)ADDR(env, outTotalHits));
  free(ar);
  free(nr);
  free(af);
  free(ns);
  free((void*)so);
  return fail(env, rc);
}
/* searchBoolAggsSortedHits for query trees, phrases and wide batches: the tree and phrase buffers as searchTreePhrases */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchTreeAggs(
    JNIEnv* env, jclass c, jlong ix, jobject clauses, jint nClauses, jobject nodes, jint nNodes, jobject phrases, jint nPhrases,
    jobject phraseTerms, jint nPhraseTerms, jobject queries, jint nq, jint topK, jint flags, jobject aggs, jint nAggs,
    jobjectArray aggOut, jobject nested, jint nNested, jobjectArray nestedOut, jobjectArray sortOrders, jobjectArray sortValues,
    jobject aggFilters, jobjectArray filterValues, jobject filterClauses, jint nFilterClauses, jobject filterQueries,
    jint nFilterQueries, jobject outDocs, jobject outScores, jobject outCounts, jobject outTotalHits) {
  nrtgpu_aggregation_result* ar = NULL;
  nrtgpu_nested_result* nr = NULL;
  nrtgpu_agg_filter* af = NULL;
  nrtgpu_nested_sort* ns = NULL;
  const nrtgpu_sort_order** so = NULL;
  int rc = agg_results(env, aggOut, nAggs, nestedOut, nNested, &ar, &nr);
  if (!rc) rc = agg_filter_records(env, aggFilters, filterValues, nAggs, &af);
  if (!rc) rc = nested_sort_records(env, sortOrders, sortValues, nNested, &ns, &so);
  if (!rc)
    rc = nrtgpu_search_tree_aggs((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                 (const nrtgpu_node*)ADDR(env, nodes), nNodes, (const nrtgpu_phrase*)ADDR(env, phrases), nPhrases,
                                 (const nrtgpu_phrase_term*)ADDR(env, phraseTerms), nPhraseTerms,
                                 (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                 (const nrtgpu_aggregation*)ADDR(env, aggs), nAggs, ar,
                                 (const nrtgpu_nested_aggregation*)ADDR(env, nested), nNested, nr, ns, af,
                                 (const nrtgpu_clause*)ADDR(env, filterClauses), nFilterClauses,
                                 (const nrtgpu_query*)ADDR(env, filterQueries), nFilterQueries, NULL,
                                 (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores),
                                 (int32_t*)ADDR(env, outCounts), (int64_t*)ADDR(env, outTotalHits));
  free(ar);
  free(nr);
  free(af);
  free(ns);
  free((void*)so);
  return fail(env, rc);
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_fetchColumns(
    JNIEnv* env, jclass c, jlong ix, jobject colIds, jint nCols, jobject docs, jint n, jobject outValues, jobject outHas) {
  return fail(env, nrtgpu_fetch_columns((nrtgpu_index*)(intptr_t)ix, (const int32_t*)ADDR(env, colIds), nCols,
                                        (const int32_t*)ADDR(env, docs), n, NULL, (int64_t*)ADDR(env, outValues),
                                        (uint8_t*)ADDR(env, outHas)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_indexSetLiveDocs(JNIEnv* env, jclass c, jlong ix, jobject live) {
  return fail(env, nrtgpu_index_set_live_docs((nrtgpu_index*)(intptr_t)ix, (const uint8_t*)ADDR(env, live)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_indexUpdateStats(
    JNIEnv* env, jclass c, jlong ix, jobject termDf, jobject fieldDocCount, jobject fieldSumTtf) {
  return fail(env, nrtgpu_index_update_stats((nrtgpu_index*)(intptr_t)ix, (const int64_t*)ADDR(env, termDf),
                                             (const int64_t*)ADDR(env, fieldDocCount), (const int64_t*)ADDR(env, fieldSumTtf)));
}
/* packed sorted records (nrtgpu_sorted_packed_words): dRecord / dRecords / dOutRecord are DEVICE addresses (the buffers a
 * multi-GPU step all-gathers), fields a direct ByteBuffer of nFields nrtgpu_sort_field */
JNIEXPORT jlong JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_sortedPackedWords(JNIEnv* env, jclass c, jint nq, jint topK, jint nFields) {
  return (jlong)nrtgpu_sorted_packed_words(nq, topK, nFields);
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searchSortedFieldsPacked(
    JNIEnv* env, jclass c, jlong ix, jlong order, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK, jint flags,
    jobject afterValues, jobject limits, jlong dRecord) {
  return fail(env, nrtgpu_search_sorted_fields_packed((nrtgpu_index*)(intptr_t)ix, (const nrtgpu_sort_order*)(intptr_t)order,
                                                      (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                                      (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                                      (const int64_t*)ADDR(env, afterValues),
                                                      (const nrtgpu_search_limits*)ADDR(env, limits), NULL, (int32_t*)(intptr_t)dRecord));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_mergeSortedPacked(
    JNIEnv* env, jclass c, jlong ctx, jobject fields, jint nFields, jint nLists, jint nq, jint topK, jlong dRecords, jlong dOutRecord) {
  return fail(env, nrtgpu_merge_sorted_packed((nrtgpu_ctx*)(intptr_t)ctx, (const nrtgpu_sort_field*)ADDR(env, fields), nFields, nLists,
                                              nq, topK, (const int32_t*)(intptr_t)dRecords, (int32_t*)(intptr_t)dOutRecord, NULL));
}
/* searchers over the leaves of one reader version: orders = a direct ByteBuffer of nOrders sort order handles (int64 each) */
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searcherSearchSortedFields(
    JNIEnv* env, jclass c, jlong s, jobject orders, jint nOrders, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK,
    jint flags, jobject afterValues, jobject limits, jobject outDocs, jobject outSortValues, jobject outCounts, jobject outTotalHits,
    jobject outRelation, jobject outHitTimeout, jobject outTerminatedEarly) {
  return fail(env, nrtgpu_searcher_search_sorted_fields((nrtgpu_searcher*)(intptr_t)s, (const nrtgpu_sort_order* const*)ADDR(env, orders),
                                                        nOrders, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                                        (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                                        (const int64_t*)ADDR(env, afterValues),
                                                        (const nrtgpu_search_limits*)ADDR(env, limits), NULL, (int32_t*)ADDR(env, outDocs),
                                                        (int64_t*)ADDR(env, outSortValues), (int32_t*)ADDR(env, outCounts),
                                                        (int64_t*)ADDR(env, outTotalHits), (uint8_t*)ADDR(env, outRelation),
                                                        (uint8_t*)ADDR(env, outHitTimeout), (uint8_t*)ADDR(env, outTerminatedEarly)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searcherSearchTreePhrases(
    JNIEnv* env, jclass c, jlong s, jobject clauses, jint nClauses, jobject nodes, jint nNodes, jobject phrases, jint nPhrases,
    jobject phraseTerms, jint nPhraseTerms, jobject queries, jint nq, jint topK, jint totalHitsThreshold, jint flags,
    jobject limits, jobject outDocs, jobject outScores, jobject outCounts, jobject outTotalHits, jobject outRelation,
    jobject outHitTimeout, jobject outTerminatedEarly) {
  return fail(env, nrtgpu_searcher_search_tree_phrases((nrtgpu_searcher*)(intptr_t)s, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                                       (const nrtgpu_node*)ADDR(env, nodes), nNodes,
                                                       (const nrtgpu_phrase*)ADDR(env, phrases), nPhrases,
                                                       (const nrtgpu_phrase_term*)ADDR(env, phraseTerms), nPhraseTerms,
                                                       (const nrtgpu_query*)ADDR(env, queries), nq, topK, totalHitsThreshold, flags,
                                                       (const nrtgpu_search_limits*)ADDR(env, limits), NULL,
                                                       (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores),
                                                       (int32_t*)ADDR(env, outCounts), (int64_t*)ADDR(env, outTotalHits),
                                                       (uint8_t*)ADDR(env, outRelation), (uint8_t*)ADDR(env, outHitTimeout),
                                                       (uint8_t*)ADDR(env, outTerminatedEarly)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searcherSearchKnn(
    JNIEnv* env, jclass c, jlong s, jobject queries, jint nq, jint k, jobject boosts, jobject filter, jobject outDocs,
    jobject outScores, jobject outCounts) {
  return fail(env, nrtgpu_searcher_search_knn((nrtgpu_searcher*)(intptr_t)s, (const float*)ADDR(env, queries), nq, k,
                                              (const float*)ADDR(env, boosts), (const uint8_t*)ADDR(env, filter), NULL,
                                              (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores), (int32_t*)ADDR(env, outCounts)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searcherSearchKnnFiltered(
    JNIEnv* env, jclass c, jlong s, jobject queries, jint nq, jint k, jobject boosts, jobject filterClauses,
    jint nFilterClauses, jobject filters, jint nFilters, jobject filterOf, jobject outDocs, jobject outScores, jobject outCounts) {
  return fail(env, nrtgpu_searcher_search_knn_filtered((nrtgpu_searcher*)(intptr_t)s, (const float*)ADDR(env, queries), nq, k,
                                                       (const float*)ADDR(env, boosts), (const nrtgpu_clause*)ADDR(env, filterClauses),
                                                       nFilterClauses, (const nrtgpu_query*)ADDR(env, filters), nFilters,
                                                       (const int32_t*)ADDR(env, filterOf), NULL, (int32_t*)ADDR(env, outDocs),
                                                       (float*)ADDR(env, outScores), (int32_t*)ADDR(env, outCounts)));
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searcherSearchBoolAggsNested(
    JNIEnv* env, jclass c, jlong s, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK, jint flags,
    jobject aggs, jint nAggs, jobjectArray aggOut, jobject nested, jint nNested, jobjectArray nestedOut, jobject outDocs,
    jobject outScores, jobject outCounts, jobject outTotalHits) {
  nrtgpu_aggregation_result* ar = NULL;
  nrtgpu_nested_result* nr = NULL;
  int rc = agg_results(env, aggOut, nAggs, nestedOut, nNested, &ar, &nr);
  if (!rc)
    rc = nrtgpu_searcher_search_bool_aggs_nested((nrtgpu_searcher*)(intptr_t)s, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                                 (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                                 (const nrtgpu_aggregation*)ADDR(env, aggs), nAggs, ar,
                                                 (const nrtgpu_nested_aggregation*)ADDR(env, nested), nNested, nr, NULL,
                                                 (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores),
                                                 (int32_t*)ADDR(env, outCounts), (int64_t*)ADDR(env, outTotalHits));
  free(ar);
  free(nr);
  return fail(env, rc);
}

JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searcherSearchBoolAggsFiltered(
    JNIEnv* env, jclass c, jlong s, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK, jint flags,
    jobject aggs, jint nAggs, jobjectArray aggOut, jobject nested, jint nNested, jobjectArray nestedOut, jobject aggFilters,
    jobjectArray filterValues, jobject filterClauses, jint nFilterClauses, jobject filterQueries, jint nFilterQueries,
    jobject outDocs, jobject outScores, jobject outCounts, jobject outTotalHits) {
  nrtgpu_aggregation_result* ar = NULL;
  nrtgpu_nested_result* nr = NULL;
  nrtgpu_agg_filter* af = NULL;
  int rc = agg_results(env, aggOut, nAggs, nestedOut, nNested, &ar, &nr);
  if (!rc) rc = agg_filter_records(env, aggFilters, filterValues, nAggs, &af);
  if (!rc)
    rc = nrtgpu_searcher_search_bool_aggs_filtered((nrtgpu_searcher*)(intptr_t)s, (const nrtgpu_clause*)ADDR(env, clauses),
                                                   nClauses, (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                                   (const nrtgpu_aggregation*)ADDR(env, aggs), nAggs, ar,
                                                   (const nrtgpu_nested_aggregation*)ADDR(env, nested), nNested, nr, af,
                                                   (const nrtgpu_clause*)ADDR(env, filterClauses), nFilterClauses,
                                                   (const nrtgpu_query*)ADDR(env, filterQueries), nFilterQueries, NULL,
                                                   (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores),
                                                   (int32_t*)ADDR(env, outCounts), (int64_t*)ADDR(env, outTotalHits));
  free(ar);
  free(nr);
  free(af);
  return fail(env, rc);
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searcherSearchBoolAggsSortedHits(
    JNIEnv* env, jclass c, jlong s, jobject clauses, jint nClauses, jobject queries, jint nq, jint topK, jint flags,
    jobject aggs, jint nAggs, jobjectArray aggOut, jobject nested, jint nNested, jobjectArray nestedOut, jobjectArray sortOrders,
    jobjectArray sortValues, jobject aggFilters, jobjectArray filterValues, jobject filterClauses, jint nFilterClauses,
    jobject filterQueries, jint nFilterQueries, jobject outDocs, jobject outScores, jobject outCounts, jobject outTotalHits) {
  nrtgpu_aggregation_result* ar = NULL;
  nrtgpu_nested_result* nr = NULL;
  nrtgpu_agg_filter* af = NULL;
  nrtgpu_nested_sort* ns = NULL;
  const nrtgpu_sort_order** so = NULL;
  int rc = agg_results(env, aggOut, nAggs, nestedOut, nNested, &ar, &nr);
  if (!rc) rc = agg_filter_records(env, aggFilters, filterValues, nAggs, &af);
  if (!rc) rc = nested_sort_records(env, sortOrders, sortValues, nNested, &ns, &so);
  if (!rc)
    rc = nrtgpu_searcher_search_bool_aggs_sorted_hits((nrtgpu_searcher*)(intptr_t)s, (const nrtgpu_clause*)ADDR(env, clauses),
                                                      nClauses, (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                                      (const nrtgpu_aggregation*)ADDR(env, aggs), nAggs, ar,
                                                      (const nrtgpu_nested_aggregation*)ADDR(env, nested), nNested, nr, ns, af,
                                                      (const nrtgpu_clause*)ADDR(env, filterClauses), nFilterClauses,
                                                      (const nrtgpu_query*)ADDR(env, filterQueries), nFilterQueries, NULL,
                                                      (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores),
                                                      (int32_t*)ADDR(env, outCounts), (int64_t*)ADDR(env, outTotalHits));
  free(ar);
  free(nr);
  free(af);
  free(ns);
  free((void*)so);
  return fail(env, rc);
}

JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_searcherSearchTreeAggs(
    JNIEnv* env, jclass c, jlong s, jobject clauses, jint nClauses, jobject nodes, jint nNodes, jobject phrases, jint nPhrases,
    jobject phraseTerms, jint nPhraseTerms, jobject queries, jint nq, jint topK, jint flags, jobject aggs, jint nAggs,
    jobjectArray aggOut, jobject nested, jint nNested, jobjectArray nestedOut, jobjectArray sortOrders, jobjectArray sortValues,
    jobject aggFilters, jobjectArray filterValues, jobject filterClauses, jint nFilterClauses, jobject filterQueries,
    jint nFilterQueries, jobject outDocs, jobject outScores, jobject outCounts, jobject outTotalHits) {
  nrtgpu_aggregation_result* ar = NULL;
  nrtgpu_nested_result* nr = NULL;
  nrtgpu_agg_filter* af = NULL;
  nrtgpu_nested_sort* ns = NULL;
  const nrtgpu_sort_order** so = NULL;
  int rc = agg_results(env, aggOut, nAggs, nestedOut, nNested, &ar, &nr);
  if (!rc) rc = agg_filter_records(env, aggFilters, filterValues, nAggs, &af);
  if (!rc) rc = nested_sort_records(env, sortOrders, sortValues, nNested, &ns, &so);
  if (!rc)
    rc = nrtgpu_searcher_search_tree_aggs((nrtgpu_searcher*)(intptr_t)s, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                          (const nrtgpu_node*)ADDR(env, nodes), nNodes, (const nrtgpu_phrase*)ADDR(env, phrases),
                                          nPhrases, (const nrtgpu_phrase_term*)ADDR(env, phraseTerms), nPhraseTerms,
                                          (const nrtgpu_query*)ADDR(env, queries), nq, topK, flags,
                                          (const nrtgpu_aggregation*)ADDR(env, aggs), nAggs, ar,
                                          (const nrtgpu_nested_aggregation*)ADDR(env, nested), nNested, nr, ns, af,
                                          (const nrtgpu_clause*)ADDR(env, filterClauses), nFilterClauses,
                                          (const nrtgpu_query*)ADDR(env, filterQueries), nFilterQueries, NULL,
                                          (int32_t*)ADDR(env, outDocs), (float*)ADDR(env, outScores),
                                          (int32_t*)ADDR(env, outCounts), (int64_t*)ADDR(env, outTotalHits));
  free(ar);
  free(nr);
  free(af);
  free(ns);
  free((void*)so);
  return fail(env, rc);
}

/* micro-batcher: one per searcher version; submit blocks the calling gRPC handler thread until its batch is back.
 * diag: 24-byte direct buffer laid out as nrtgpu_diagnostics, or null */
JNIEXPORT jlong JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_batcherCreate(JNIEnv* env, jclass c, jlong ix, jint maxBatch, jint maxWaitUs) {
  nrtgpu_batcher* b = NULL;
  if (fail(env, nrtgpu_batcher_create((nrtgpu_index*)(intptr_t)ix, maxBatch, maxWaitUs, &b))) return 0;
  return (jlong)(intptr_t)b;
}
JNIEXPORT jint JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_batcherSubmit(
    JNIEnv* env, jclass c, jlong b, jobject clauses, jint nClauses, jint minShouldMatch, jint topK, jint totalHitsThreshold,
    jobject outDocs, jobject outScores, jobject outCount, jobject outTotalHits, jobject outRelation, jobject diag) {
  return fail(env, nrtgpu_batcher_submit((nrtgpu_batcher*)(intptr_t)b, (const nrtgpu_clause*)ADDR(env, clauses), nClauses,
                                         minShouldMatch, topK, totalHitsThreshold, (int32_t*)ADDR(env, outDocs),
                                         (float*)ADDR(env, outScores), (int32_t*)ADDR(env, outCount),
                                         (int64_t*)ADDR(env, outTotalHits), (uint8_t*)ADDR(env, outRelation),
                                         (nrtgpu_diagnostics*)ADDR(env, diag)));
}
JNIEXPORT void JNICALL Java_com_yelp_nrtsearch_server_gpu_NrtGpu_batcherClose(JNIEnv* env, jclass c, jlong b) {
  nrtgpu_batcher_close((nrtgpu_batcher*)(intptr_t)b);
}
