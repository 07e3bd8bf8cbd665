package com.yelp.nrtsearch.server.gpu;

import java.nio.ByteBuffer;

/** JNI binding of include/nrtgpu.h (one native method per C entry point; direct buffers only). */
public final class NrtGpu {
  static {
    System.loadLibrary("nrtgpu_jni");
  }

  private NrtGpu() {}

  public static native long init(int device);

  public static native void shutdown(long ctx);

  public static native long indexBuild(long ctx, ByteBuffer shardDesc);

  public static native void indexClose(long index);

  public static native int searchBool(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK,
      int totalHitsThreshold, int flags, ByteBuffer outDocs, ByteBuffer outScores,
      ByteBuffer outCounts, ByteBuffer outTotalHits, ByteBuffer outRelation);

  public static native int searchKnn(
      long index, ByteBuffer queries, int nq, int k, ByteBuffer boosts, ByteBuffer filter,
      ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCounts);

  /** kNN with one filter query per query vector (KnnQuery.filter); filterOf[q] indexes filters, -1 = none. */
  public static native int searchKnnFiltered(
      long index, ByteBuffer queries, int nq, int k, ByteBuffer boosts, ByteBuffer filterClauses,
      int nFilterClauses, ByteBuffer filters, int nFilters, ByteBuffer filterOf, ByteBuffer outDocs,
      ByteBuffer outScores, ByteBuffer outCounts);

  public static native int blendRrf(
      long ctx, int nRetrievers, int nq, int topIn, ByteBuffer docs, ByteBuffer counts,
      ByteBuffer boosts, int rankConstant, int topOut, ByteBuffer outDocs, ByteBuffer outScores,
      ByteBuffer outCounts, ByteBuffer outTotal);

  public static native int rescoreCombine(
      long ctx, int nq, int nHits, ByteBuffer counts, ByteBuffer docs, ByteBuffer scores,
      ByteBuffer secondMatches, ByteBuffer secondScores, double queryWeight, double rescoreWeight);

  /** limits = nrtgpu_search_limits or null; outHitTimeout / outTerminatedEarly may be null. */
  public static native int searchBoolEx(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK,
      int totalHitsThreshold, int flags, ByteBuffer limits, ByteBuffer outDocs,
      ByteBuffer outScores, ByteBuffer outCounts, ByteBuffer outTotalHits, ByteBuffer outRelation,
      ByteBuffer outHitTimeout, ByteBuffer outTerminatedEarly);

  /**
   * Query trees (nested BooleanQuery / DisjunctionMaxQuery / ConstantScoreQuery / MinScoreQuery / NestedQuery): nodes =
   * nrtgpu_node[nNodes] (28 bytes each: int kind (0 BOOL, 1 DISMAX, 3 CONSTANT, 4 MIN_SCORE, 6 NESTED), clauseBegin,
   * clauseEnd, minShouldMatch (NESTED: the score mode, 0 NONE 1 AVG 2 MAX 3 MIN 4 SUM), float tieBreaker, boost,
   * minScore), referenced by clauses of kind 3 (NODE); a NESTED node holds one MUST clause, the child query
   * {FILTER _nested_path:path, MUST child}, and needs addParents; otherwise as searchBoolEx, which it is with nNodes == 0.
   */
  public static native int searchTree(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer nodes, int nNodes, ByteBuffer queries, int nq,
      int topK, int totalHitsThreshold, int flags, ByteBuffer limits, ByteBuffer outDocs, ByteBuffer outScores,
      ByteBuffer outCounts, ByteBuffer outTotalHits, ByteBuffer outRelation, ByteBuffer outHitTimeout,
      ByteBuffer outTerminatedEarly);

  /**
   * Term positions of the image: positions = nPositions int32, posting after posting in the build's CSR order, the freq
   * positions of each posting ascending (PostingsEnum.nextPosition() with PostingsEnum.POSITIONS).
   */
  public static native int addPositions(long index, ByteBuffer positions, long nPositions);

  /**
   * The parent docs of the image's blocks (NESTED nodes): the docs of term rootTerm (_nested_path:_root), kept as a
   * bitset on the device across live-doc and statistics refreshes.
   */
  public static native int addParents(long index, int rootTerm);

  /**
   * Keyword columns of an image, read per leaf from SortedDocValues / SortedSetDocValues when the image is built: column k
   * has nTerms[k] terms (termBytes, termOffsets int64[nTerms + 1], ascending in BytesRef order) and ords int32 per doc
   * (SORTED, -1: no value) or int32 per value with docOffsets int64[maxDoc + 1] (SORTED_SET, multiValued[k] = 1). Once per
   * image. A TermsCollector on the field is then an nrtgpu_aggregation with value_type 3 naming column k.
   */
  public static native int addKeywordColumns(long index, int[] nTerms, int[] multiValued, ByteBuffer[] termBytes,
      ByteBuffer[] termOffsets, ByteBuffer[] ords, ByteBuffer[] docOffsets);

  /** The bytes of term ord of keyword column `column` into out (at most cap); returns its length (bucket keys -> BytesRef). */
  public static native int keywordTerm(long index, int column, int ord, ByteBuffer out, int cap);

  /** keywordTerm for a searcher's reader-wide ordinals; ord -1 returns the number of reader-wide terms. */
  public static native int searcherKeywordTerm(long searcher, int column, int ord, ByteBuffer out, int cap);

  /** nrtgpu_sort_field.kind of a keyword sort field (AtomFieldDef.getSortField); missing_value 0 STRING_FIRST, 1 STRING_LAST. */
  public static final int SORT_KEYWORD = 5;
  /** nrtgpu_sort_field.selector (SortedSetSelector.Type); MIDDLE_* only on a SORTED_SET keyword field. */
  public static final int SELECT_MIN = 0, SELECT_MAX = 1, SELECT_MIDDLE_MIN = 2, SELECT_MIDDLE_MAX = 3;

  /**
   * The sort code of a keyword term (len bytes of the direct buffer term) in keyword column `column` of an image: 2i + 2
   * for its term i, 2i + 1 for a term it does not hold. A LastHitInfo string becomes a keyword field's after value this way
   * (NULL_SORT_VALUE is 0); FieldDoc values c map back to terms with keywordTerm(c / 2 - 1).
   */
  public static native long keywordSeek(long index, int column, ByteBuffer term, int len);

  /** keywordSeek in a searcher's reader-wide dictionary (the codes of searcherSearchSortedFields). */
  public static native long searcherKeywordSeek(long searcher, int column, ByteBuffer term, int len);

  /** Keyword range clauses (clause kind 5, KEYWORD_RANGE): flags of keywordRange. */
  public static final int KEYWORD_NO_LOWER = 1, KEYWORD_NO_UPPER = 2, KEYWORD_LOWER_EXCLUSIVE = 4, KEYWORD_UPPER_EXCLUSIVE = 8,
      KEYWORD_PREFIX = 16;

  /**
   * The code range of a TermRangeQuery or PrefixQuery on an atom field: out (two longs) receives [lo, hi] for a KEYWORD_RANGE
   * clause, in the image's dictionary (searcher 0) or the searcher's reader-wide one. The bounds are the field's normalized
   * bytes (AtomFieldDef.normalize).
   */
  public static native int keywordRange(long index, long searcher, int column, ByteBuffer lower, int lowerLen, ByteBuffer upper,
                                        int upperLen, int flags, ByteBuffer out);

  /**
   * Query trees with PhraseQuery leaves: phrases = nrtgpu_phrase[nPhrases] referenced by clauses of kind 4 (PHRASE)
   * or kind 6 (MULTI_PHRASE: MultiPhraseQuery, match_phrase_prefix with its prefix expanded by the caller; terms that
   * share a position are alternatives), phraseTerms = nrtgpu_phrase_term[nPhraseTerms] (term id, position); otherwise
   * as searchTree, which it is with nPhrases == 0.
   */
  public static native int searchTreePhrases(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer nodes, int nNodes, ByteBuffer phrases, int nPhrases,
      ByteBuffer phraseTerms, int nPhraseTerms, ByteBuffer queries, int nq, int topK, int totalHitsThreshold, int flags,
      ByteBuffer limits, ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCounts, ByteBuffer outTotalHits,
      ByteBuffer outRelation, ByteBuffer outHitTimeout, ByteBuffer outTerminatedEarly);

  public static native int searchSorted(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK, int flags,
      ByteBuffer sort, ByteBuffer limits, ByteBuffer outDocs, ByteBuffer outSortValues,
      ByteBuffer outCounts, ByteBuffer outTotalHits, ByteBuffer outRelation,
      ByteBuffer outHitTimeout, ByteBuffer outTerminatedEarly);

  /** fields = nFields nrtgpu_sort_field; the order handle is written to outOrder (8 bytes). */
  public static native int sortOrderCreate(long index, ByteBuffer fields, int nFields, ByteBuffer outOrder);

  public static native long sortOrderDeviceBytes(long order);

  public static native int sortOrderClose(long order);

  /** afterValues = nq * nFields FieldDoc values (or null); outSortValues = nq * topK * nFields. */
  public static native int searchSortedFields(
      long index, long order, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK,
      int flags, ByteBuffer afterValues, ByteBuffer limits, ByteBuffer outDocs, ByteBuffer outSortValues,
      ByteBuffer outCounts, ByteBuffer outTotalHits, ByteBuffer outRelation,
      ByteBuffer outHitTimeout, ByteBuffer outTerminatedEarly);

  public static native int scoreDocs(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int nHits,
      ByteBuffer docs, ByteBuffer counts, ByteBuffer outMatches, ByteBuffer outScores);

  /**
   * QueryRescorer second pass (scoreDocsTree) and whole rescore (rescoreQueryTree, docs / scores rescored in place) for a
   * rescore query that is a query tree or holds phrases; the tree and phrase buffers are laid out as for searchTreePhrases,
   * the hit buffers as for scoreDocs.
   */
  public static native int scoreDocsTree(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer nodes, int nNodes, ByteBuffer phrases, int nPhrases,
      ByteBuffer phraseTerms, int nPhraseTerms, ByteBuffer queries, int nq, int nHits, ByteBuffer docs, ByteBuffer counts,
      ByteBuffer outMatches, ByteBuffer outScores);

  public static native int rescoreQueryTree(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer nodes, int nNodes, ByteBuffer phrases, int nPhrases,
      ByteBuffer phraseTerms, int nPhraseTerms, ByteBuffer queries, int nq, int nHits, ByteBuffer counts, int window,
      double queryWeight, double rescoreWeight, ByteBuffer docs, ByteBuffer scores, ByteBuffer outCounts);

  /**
   * Additional collectors with nested collectors (nrtgpu_search_bool_aggs_nested): aggs = nAggs nrtgpu_aggregation, nested =
   * nNested nrtgpu_nested_aggregation; aggOut holds 6 buffers (or null) per aggregation in nrtgpu_aggregation_result field
   * order, nestedOut 5 per nested collector in nrtgpu_nested_result field order.
   */
  public static native int searchBoolAggsNested(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK, int flags, ByteBuffer aggs,
      int nAggs, ByteBuffer[] aggOut, ByteBuffer nested, int nNested, ByteBuffer[] nestedOut, ByteBuffer outDocs,
      ByteBuffer outScores, ByteBuffer outCounts, ByteBuffer outTotalHits);

  public static native int fetchColumns(
      long index, ByteBuffer colIds, int nCols, ByteBuffer docs, int n, ByteBuffer outValues,
      ByteBuffer outHas);

  public static native int indexSetLiveDocs(long index, ByteBuffer liveDocs);

  public static native int indexUpdateStats(
      long index, ByteBuffer termDf, ByteBuffer fieldDocCount, ByteBuffer fieldSumTtf);

  /** Size in int32 words of a packed sorted record (include/nrtgpu.h nrtgpu_sorted_packed_words). */
  public static native long sortedPackedWords(int nq, int topK, int nFields);

  /** searchSortedFields with the results left in the DEVICE record at address dRecord. */
  public static native int searchSortedFieldsPacked(
      long index, long order, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK,
      int flags, ByteBuffer afterValues, ByteBuffer limits, long dRecord);

  /** TopFieldDocs.merge of nLists DEVICE sorted records at dRecords into dOutRecord; fields = the Sort's nrtgpu_sort_field. */
  public static native int mergeSortedPacked(
      long ctx, ByteBuffer fields, int nFields, int nLists, int nq, int topK, long dRecords, long dOutRecord);

  /** Sorted search over the leaves of a searcher: orders = one sort order handle (int64) per leaf, all of one Sort. */
  public static native int searcherSearchSortedFields(
      long searcher, ByteBuffer orders, int nOrders, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq,
      int topK, int flags, ByteBuffer afterValues, ByteBuffer limits, ByteBuffer outDocs, ByteBuffer outSortValues,
      ByteBuffer outCounts, ByteBuffer outTotalHits, ByteBuffer outRelation, ByteBuffer outHitTimeout,
      ByteBuffer outTerminatedEarly);

  /** searchTreePhrases over the leaves of a searcher. */
  public static native int searcherSearchTreePhrases(
      long searcher, ByteBuffer clauses, int nClauses, ByteBuffer nodes, int nNodes, ByteBuffer phrases, int nPhrases,
      ByteBuffer phraseTerms, int nPhraseTerms, ByteBuffer queries, int nq, int topK, int totalHitsThreshold, int flags,
      ByteBuffer limits, ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCounts, ByteBuffer outTotalHits,
      ByteBuffer outRelation, ByteBuffer outHitTimeout, ByteBuffer outTerminatedEarly);

  /** searchKnn over the leaves of a searcher; filter = one byte per global doc id (or null). */
  public static native int searcherSearchKnn(
      long searcher, ByteBuffer queries, int nq, int k, ByteBuffer boosts, ByteBuffer filter,
      ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCounts);

  /** searchKnnFiltered over the leaves of a searcher. */
  public static native int searcherSearchKnnFiltered(
      long searcher, ByteBuffer queries, int nq, int k, ByteBuffer boosts, ByteBuffer filterClauses,
      int nFilterClauses, ByteBuffer filters, int nFilters, ByteBuffer filterOf, ByteBuffer outDocs,
      ByteBuffer outScores, ByteBuffer outCounts);

  /**
   * searchBoolAggsNested over the leaves of a searcher (nNested may be 0): terms buckets counted by value across the
   * leaves, nested top hits chosen per reader-wide bucket; the same buffers as searchBoolAggsNested.
   */
  public static native int searcherSearchBoolAggsNested(
      long searcher, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK, int flags, ByteBuffer aggs,
      int nAggs, ByteBuffer[] aggOut, ByteBuffer nested, int nNested, ByteBuffer[] nestedOut, ByteBuffer outDocs,
      ByteBuffer outScores, ByteBuffer outCounts, ByteBuffer outTotalHits);

  /**
   * Additional collectors with filter collectors (nrtgpu_search_bool_aggs_filtered): the buffers of searchBoolAggsNested, plus
   * aggFilters = nAggs nrtgpu_agg_filter (their values fields are ignored), filterValues = one int64 buffer (or null) per
   * aggregation holding a VALUE_SET filter's set, and the filter queries (filterClauses / filterQueries, the clause format
   * of searchBool). A FILTER aggregation's docCount comes back in its bucket_counts buffer.
   */
  public static native int searchBoolAggsFiltered(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK, int flags, ByteBuffer aggs,
      int nAggs, ByteBuffer[] aggOut, ByteBuffer nested, int nNested, ByteBuffer[] nestedOut, ByteBuffer aggFilters,
      ByteBuffer[] filterValues, ByteBuffer filterClauses, int nFilterClauses, ByteBuffer filterQueries, int nFilterQueries,
      ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCounts, ByteBuffer outTotalHits);

  /** searchBoolAggsFiltered over the leaves of a searcher: docCount and everything under a filter are reader-wide. */
  public static native int searcherSearchBoolAggsFiltered(
      long searcher, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK, int flags, ByteBuffer aggs,
      int nAggs, ByteBuffer[] aggOut, ByteBuffer nested, int nNested, ByteBuffer[] nestedOut, ByteBuffer aggFilters,
      ByteBuffer[] filterValues, ByteBuffer filterClauses, int nFilterClauses, ByteBuffer filterQueries, int nFilterQueries,
      ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCounts, ByteBuffer outTotalHits);

  /**
   * searchBoolAggsFiltered plus sorted top hits (TopHitsCollector.querySort; include/nrtgpu.h
   * nrtgpu_search_bool_aggs_sorted_hits): sortOrders[j] the sort-order handles of nested collector j (one, from
   * sortOrderCreate on this index; null: by score), sortValues[j] a direct buffer for its FieldDoc values (or null). A
   * top-level TopHitsCollector is the nested top hits of a FILTER aggregation with a match-all filter query.
   */
  public static native int searchBoolAggsSortedHits(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK, int flags, ByteBuffer aggs,
      int nAggs, ByteBuffer[] aggOut, ByteBuffer nested, int nNested, ByteBuffer[] nestedOut, long[][] sortOrders,
      ByteBuffer[] sortValues, ByteBuffer aggFilters, ByteBuffer[] filterValues, ByteBuffer filterClauses, int nFilterClauses,
      ByteBuffer filterQueries, int nFilterQueries, ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCounts,
      ByteBuffer outTotalHits);

  /** searchBoolAggsSortedHits over the leaves of a searcher: sortOrders[j] holds one order per leaf, in leaf order. */
  public static native int searcherSearchBoolAggsSortedHits(
      long searcher, ByteBuffer clauses, int nClauses, ByteBuffer queries, int nq, int topK, int flags, ByteBuffer aggs,
      int nAggs, ByteBuffer[] aggOut, ByteBuffer nested, int nNested, ByteBuffer[] nestedOut, long[][] sortOrders,
      ByteBuffer[] sortValues, ByteBuffer aggFilters, ByteBuffer[] filterValues, ByteBuffer filterClauses, int nFilterClauses,
      ByteBuffer filterQueries, int nFilterQueries, ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCounts,
      ByteBuffer outTotalHits);

  /**
   * searchBoolAggsSortedHits for the queries of searchTreePhrases (include/nrtgpu.h nrtgpu_search_tree_aggs): nested
   * BooleanQuery / DisjunctionMaxQuery, PhraseQuery leaves and flat batches of more than 4 term clauses or topK > 512, their
   * collectors run by the window engine. The tree and phrase buffers as searchTreePhrases (nNodes / nPhrases may be 0), the
   * collector arguments as searchBoolAggsSortedHits.
   */
  public static native int searchTreeAggs(
      long index, ByteBuffer clauses, int nClauses, ByteBuffer nodes, int nNodes, ByteBuffer phrases, int nPhrases,
      ByteBuffer phraseTerms, int nPhraseTerms, ByteBuffer queries, int nq, int topK, int flags, ByteBuffer aggs, int nAggs,
      ByteBuffer[] aggOut, ByteBuffer nested, int nNested, ByteBuffer[] nestedOut, long[][] sortOrders, ByteBuffer[] sortValues,
      ByteBuffer aggFilters, ByteBuffer[] filterValues, ByteBuffer filterClauses, int nFilterClauses, ByteBuffer filterQueries,
      int nFilterQueries, ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCounts, ByteBuffer outTotalHits);

  /** searchTreeAggs over the leaves of a searcher: sortOrders[j] holds one order per leaf, in leaf order. */
  public static native int searcherSearchTreeAggs(
      long searcher, ByteBuffer clauses, int nClauses, ByteBuffer nodes, int nNodes, ByteBuffer phrases, int nPhrases,
      ByteBuffer phraseTerms, int nPhraseTerms, ByteBuffer queries, int nq, int topK, int flags, ByteBuffer aggs, int nAggs,
      ByteBuffer[] aggOut, ByteBuffer nested, int nNested, ByteBuffer[] nestedOut, long[][] sortOrders, ByteBuffer[] sortValues,
      ByteBuffer aggFilters, ByteBuffer[] filterValues, ByteBuffer filterClauses, int nFilterClauses, ByteBuffer filterQueries,
      int nFilterQueries, ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCounts, ByteBuffer outTotalHits);

  public static native long batcherCreate(long index, int maxBatch, int maxWaitUs);

  /** Blocks until the batch this request rode in is back; diag = nrtgpu_diagnostics (24 bytes) or null. */
  public static native int batcherSubmit(
      long batcher, ByteBuffer clauses, int nClauses, int minShouldMatch, int topK,
      int totalHitsThreshold, ByteBuffer outDocs, ByteBuffer outScores, ByteBuffer outCount,
      ByteBuffer outTotalHits, ByteBuffer outRelation, ByteBuffer diag);

  public static native void batcherClose(long batcher);
}
