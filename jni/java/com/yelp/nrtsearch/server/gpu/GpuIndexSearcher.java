package com.yelp.nrtsearch.server.gpu;

import com.yelp.nrtsearch.server.search.MyIndexSearcher;
import java.io.IOException;
import java.nio.ByteBuffer;
import java.nio.ByteOrder;
import org.apache.lucene.index.IndexReader;
import org.apache.lucene.search.CollectorManager;
import org.apache.lucene.search.Query;
import org.apache.lucene.search.ScoreDoc;
import org.apache.lucene.search.TopDocs;
import org.apache.lucene.search.TotalHits;

/**
 * Reference-side adaptor (not built in the authoring image: no JDK / Lucene jars there). A MyIndexSearcher subclass
 * created at ShardState.ShardSearcherFactory.newSearcher (ShardState.java:506-526). search() pattern-matches the
 * rewritten Query (flat BooleanQuery of TermQuery / IndexOrDocValuesQuery range / MatchAllDocsQuery, optional
 * BoostQuery wrappers; or a tree of nested BooleanQuery / DisjunctionMaxQuery nodes over those leaves and PhraseQuery
 * leaves) and the RelevanceCollector configuration. A compiled request that carries nodes or phrases calls
 * nrtgpu_search_tree / nrtgpu_search_tree_phrases directly on the handler thread (MultiPhraseQuery and phrase-prefix
 * queries are not compiled: Lucene). Any other supported request is handed to the NATIVE
 * micro-batcher (nrtgpu_batcher_submit): the gRPC handler thread blocks while a worker thread inside libnrtgpu groups
 * the waiting requests into one batched search. Everything else, and NRTGPU_ERR_UNSUPPORTED
 * (UnsupportedOperationException), falls through to super.search(), i.e. Lucene. The image and its batcher are released
 * in close(), called after the last ShardState.release (:406-425).
 */
public class GpuIndexSearcher extends MyIndexSearcher {
  private final long gpuIndex; // nrtgpu_index* of this reader version
  private final long batcher; // nrtgpu_batcher* bound to gpuIndex
  private final GpuQueryCompiler compiler; // term -> dense id dictionary built with the image
  // nrtgpu_sort_order* of this leaf per Sort (key: its nrtgpu_sort_field records)
  private final java.util.concurrent.ConcurrentHashMap<ByteBuffer, Long> sortOrders =
      new java.util.concurrent.ConcurrentHashMap<>();

  protected GpuIndexSearcher(
      IndexReader reader,
      java.util.concurrent.Executor executor,
      long gpuIndex,
      GpuQueryCompiler compiler,
      int maxBatch,
      int maxWaitUs) {
    super(reader, executor);
    this.gpuIndex = gpuIndex;
    this.compiler = compiler;
    this.batcher = NrtGpu.batcherCreate(gpuIndex, maxBatch, maxWaitUs);
  }

  @Override
  public <C extends org.apache.lucene.search.Collector, T> T search(
      Query query, CollectorManager<C, T> collectorManager) throws IOException {
    GpuQueryCompiler.Compiled c = compiler.tryCompile(query, collectorManager);
    if (c == null) {
      return super.search(query, collectorManager); // not on the GPU path: Lucene
    }
    if (c.sortFields() != null) {
      T sorted = searchSortedFields(c);
      return sorted != null ? sorted : super.search(query, collectorManager);
    }
    if (c.numNodes() > 0 || c.numPhrases() > 0) {
      T tree = searchTree(c);
      return tree != null ? tree : super.search(query, collectorManager);
    }
    int k = c.topK();
    ByteBuffer docs = direct(4 * k), scores = direct(4 * k), count = direct(4), total = direct(8);
    ByteBuffer relation = direct(1), diag = direct(24);
    try {
      NrtGpu.batcherSubmit(
          batcher, c.clauses(), c.numClauses(), c.minShouldMatch(), k, c.totalHitsThreshold(), docs,
          scores, count, total, relation, diag);
    } catch (UnsupportedOperationException e) {
      return super.search(query, collectorManager);
    }
    int n = count.getInt(0);
    ScoreDoc[] hits = new ScoreDoc[n];
    for (int i = 0; i < n; ++i) {
      hits[i] = new ScoreDoc(docs.getInt(4 * i), scores.getFloat(4 * i));
    }
    TotalHits.Relation rel =
        relation.get(0) == 0
            ? TotalHits.Relation.EQUAL_TO
            : TotalHits.Relation.GREATER_THAN_OR_EQUAL_TO;
    // Diagnostics of the request (SearchHandler.java:261,280,321): queue_ms, search_ms, batch_size
    return c.toResult(
        new TopDocs(new TotalHits(total.getLong(0), rel), hits),
        diag.getDouble(0),
        diag.getDouble(8),
        diag.getInt(16));
  }

  /**
   * SortFieldCollector with a Sort of several fields (or a score / multi-valued field): one nrtgpu_sort_order per Sort,
   * built on first use and kept with this leaf's image (it depends on the columns only). null = UNSUPPORTED: Lucene.
   */
  private <T> T searchSortedFields(GpuQueryCompiler.Compiled c) {
    ByteBuffer fields = c.sortFields();
    int nFields = c.numSortFields(), k = c.topK();
    byte[] spec = new byte[24 * nFields];
    fields.duplicate().get(spec);
    long order;
    try {
      order =
          sortOrders.computeIfAbsent(
              java.nio.ByteBuffer.wrap(spec),
              key -> {
                ByteBuffer out = direct(8);
                NrtGpu.sortOrderCreate(gpuIndex, fields, nFields, out);
                return out.getLong(0);
              });
    } catch (UnsupportedOperationException e) {
      return null;
    }
    ByteBuffer docs = direct(4 * k), values = direct(8 * k * nFields), count = direct(4), total = direct(8);
    ByteBuffer relation = direct(1), hitTimeout = direct(1), terminated = direct(1);
    try {
      NrtGpu.searchSortedFields(
          gpuIndex, order, c.clauses(), c.numClauses(), c.queries(), 1, k, 0, c.afterValues(), c.limits(), docs,
          values, count, total, relation, hitTimeout, terminated);
    } catch (UnsupportedOperationException e) {
      return null;
    }
    int n = count.getInt(0);
    int[] hitDocs = new int[n];
    long[][] hitValues = new long[n][nFields];
    for (int i = 0; i < n; ++i) {
      hitDocs[i] = docs.getInt(4 * i);
      for (int f = 0; f < nFields; ++f) {
        hitValues[i][f] = values.getLong(8 * (i * nFields + f));
      }
    }
    TotalHits.Relation rel =
        relation.get(0) == 0
            ? TotalHits.Relation.EQUAL_TO
            : TotalHits.Relation.GREATER_THAN_OR_EQUAL_TO;
    return c.toSortedResult(
        new TotalHits(total.getLong(0), rel), hitDocs, hitValues, hitTimeout.get(0) != 0, terminated.get(0) != 0);
  }

  /**
   * A query tree (nested BooleanQuery / DisjunctionMaxQuery, PhraseQuery leaves; the micro-batcher takes flat queries
   * only): one nrtgpu_search_tree(_phrases) call for this request. null = UNSUPPORTED (past the tree limits, a sloppy
   * phrase with a repeated term): Lucene.
   */
  private <T> T searchTree(GpuQueryCompiler.Compiled c) {
    int k = c.topK();
    ByteBuffer docs = direct(4 * k), scores = direct(4 * k), count = direct(4), total = direct(8);
    ByteBuffer relation = direct(1), hitTimeout = direct(1), terminated = direct(1);
    long t0 = System.nanoTime();
    try {
      if (c.numPhrases() > 0) {
        NrtGpu.searchTreePhrases(
            gpuIndex, c.clauses(), c.numClauses(), c.nodes(), c.numNodes(), c.phrases(), c.numPhrases(), c.phraseTerms(),
            c.numPhraseTerms(), c.queries(), 1, k, c.totalHitsThreshold(), 0, c.limits(), docs, scores, count, total,
            relation, hitTimeout, terminated);
      } else {
        NrtGpu.searchTree(
            gpuIndex, c.clauses(), c.numClauses(), c.nodes(), c.numNodes(), c.queries(), 1, k, c.totalHitsThreshold(), 0,
            c.limits(), docs, scores, count, total, relation, hitTimeout, terminated);
      }
    } catch (UnsupportedOperationException e) {
      return null;
    }
    double searchMs = (System.nanoTime() - t0) / 1e6;
    int n = count.getInt(0);
    ScoreDoc[] hits = new ScoreDoc[n];
    for (int i = 0; i < n; ++i) {
      hits[i] = new ScoreDoc(docs.getInt(4 * i), scores.getFloat(4 * i));
    }
    TotalHits.Relation rel =
        relation.get(0) == 0
            ? TotalHits.Relation.EQUAL_TO
            : TotalHits.Relation.GREATER_THAN_OR_EQUAL_TO;
    return c.toResult(new TopDocs(new TotalHits(total.getLong(0), rel), hits), 0.0, searchMs, 1);
  }

  public void close() {
    for (long order : sortOrders.values()) {
      NrtGpu.sortOrderClose(order);
    }
    NrtGpu.batcherClose(batcher);
    NrtGpu.indexClose(gpuIndex);
  }

  /**
   * Appends a Lucene PhraseQuery as one nrtgpu_phrase record (into phrases) and its nrtgpu_phrase_term records (into
   * phraseTerms, starting at record index firstTerm): PhraseQuery.getTerms() mapped through termId, getPositions() and
   * getSlop() as they are. Returns the phrase's index for the PHRASE clause's id, or -1 when a term is not in the
   * dictionary (the compiler then emits a phrase of no terms: it matches nothing, as in Lucene).
   */
  public static int appendPhrase(
      org.apache.lucene.search.PhraseQuery q,
      java.util.function.ToIntFunction<org.apache.lucene.index.Term> termId,
      ByteBuffer phrases,
      int phraseIndex,
      ByteBuffer phraseTerms,
      int firstTerm) {
    org.apache.lucene.index.Term[] terms = q.getTerms();
    int[] positions = q.getPositions();
    for (int i = 0; i < terms.length; ++i) {
      int id = termId.applyAsInt(terms[i]);
      if (id < 0) {
        return -1;
      }
      phraseTerms.putInt(8 * (firstTerm + i), id).putInt(8 * (firstTerm + i) + 4, positions[i]);
    }
    phrases
        .putInt(16 * phraseIndex, firstTerm)
        .putInt(16 * phraseIndex + 4, firstTerm + terms.length)
        .putInt(16 * phraseIndex + 8, q.getSlop())
        .putInt(16 * phraseIndex + 12, 0);
    return phraseIndex;
  }

  private static ByteBuffer direct(int bytes) {
    return ByteBuffer.allocateDirect(bytes).order(ByteOrder.nativeOrder());
  }

  /** Compiles Lucene queries to nrtgpu_clause records (see INTEGRATION.md for the rules). */
  public interface GpuQueryCompiler {
    Compiled tryCompile(Query query, CollectorManager<?, ?> manager);

    interface Compiled {
      ByteBuffer clauses(); // direct, nrtgpu_clause[numClauses]

      int numClauses();

      int minShouldMatch();

      int topK();

      int totalHitsThreshold();

      <T> T toResult(TopDocs topDocs, double queueMs, double searchMs, int batchSize);

      /**
       * SortFieldCollector requests: nrtgpu_sort_field[numSortFields()], or null for relevance. A SortField of an AtomFieldDef
       * (STRING or SortedSetSortField) is kind NrtGpu.SORT_KEYWORD on the field's keyword column, its selector one of
       * NrtGpu.SELECT_*, missing_value 1 for STRING_LAST; its after value is NrtGpu.keywordSeek of the LastHitInfo string
       * (searcherKeywordSeek over several leaves), or 0 for NULL_SORT_VALUE.
       */
      default ByteBuffer sortFields() {
        return null;
      }

      default int numSortFields() {
        return 0;
      }

      default ByteBuffer queries() { // direct, one nrtgpu_query (msm of the root; has_after / after_doc, after_score)
        return null;
      }

      default ByteBuffer afterValues() { // direct, numSortFields() int64 FieldDoc values, or null
        return null;
      }

      default ByteBuffer limits() { // direct nrtgpu_search_limits, or null
        return null;
      }

      /** Query trees: nrtgpu_node[numNodes()] referenced by the NODE clauses, or null for a flat query. */
      default ByteBuffer nodes() {
        return null;
      }

      default int numNodes() {
        return 0;
      }

      /**
       * PhraseQuery leaves (clauses of kind 4): nrtgpu_phrase[numPhrases()] and nrtgpu_phrase_term[numPhraseTerms()]
       * (see appendPhrase), or null for a request without phrases.
       */
      default ByteBuffer phrases() {
        return null;
      }

      default int numPhrases() {
        return 0;
      }

      default ByteBuffer phraseTerms() {
        return null;
      }

      default int numPhraseTerms() {
        return 0;
      }

      /** TopFieldDocs from raw FieldDoc values (the compiler knows each field's type). */
      default <T> T toSortedResult(
          TotalHits totalHits, int[] docs, long[][] values, boolean hitTimeout, boolean terminatedEarly) {
        throw new UnsupportedOperationException("sorted results");
      }
    }
  }
}
