"""Wide batches: the window engine (bool_window_kernel, bool_kernel.cuh) against the exhaustive oracle.

compile_batch (csrc/batch_plan.inc) picks the engine for a WHOLE batch: one query with more than 4 term clauses, or any top_k above
512, sends every query of the batch through bool_window_kernel -- 1,048,576-doc slices of 64 windows of 16,384 docs, a
4096-key candidate buffer compacted mid-window, exact_freq_slow for tf >= 255, a dense-driver sweep for match-all and
range-led queries -- then merge_slices_kernel, and merge_pairs_kernel across leaves, at up to top_k 1024.

Every page is compared with oracle.search_compiled: equal counts, the same doc sequence, bit-identical scores, totalHits
exact when EQUAL_TO and in (threshold, exact] when GREATER_THAN_OR_EQUAL_TO. Every test first proves that its batch went
wide (assert_wide): the window engine has exactly one work item per (non-empty query, 1,048,576-doc slice), while the
probe engine splits a shard into slices of at most 524,288 docs, so on a larger shard it has more items per query."""
import numpy as np
import pytest

import oracle
from helpers import assert_same_hits, shard_from_token_docs
from nrtsearch_b200 import NrtGpuUnsupported
from nrtsearch_b200 import index as ix
from nrtsearch_b200._native import CollectionTimeoutException
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, GpuIndex, GpuIndexSearcher, GpuLeafSearcher, MatchAllDocsQuery,
                                   MinCollector, Occur, RangeQuery, RelevanceCollector, ScoreDoc, SortFieldCollector, SortType,
                                   TermQuery, compile_queries)

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
WIDE_SLICE = 64 * 16384     # bool_window_kernel: kSliceWindows * kWindowDocs
PROBE_SLICE = 512 * 1024    # probe kernel: at most slice_gran (512) granules of 1024 docs
N_MIX = 600_000             # > PROBE_SLICE: probe and window batches differ in work items


# ---------------------------------------------------------------- helpers

def n_nonempty(queries):
    """Queries plan_work gives work items: not (msm > #SHOULD, or no MUST / FILTER / SHOULD clause at all)."""
    carr, _, qarr, nq = compile_queries(queries)
    n = 0
    for i in range(nq):
        occ = [carr[c].occur for c in range(qarr[i].clause_begin, qarr[i].clause_end)]
        n_should = sum(o == Occur.SHOULD for o in occ)
        n_req = sum(o in (Occur.MUST, Occur.FILTER) for o in occ)
        n += not (qarr[i].min_should_match > n_should or (n_req == 0 and n_should == 0))
    return n


def work_items(gix, queries, k, threshold=INT_MAX):
    b = GpuIndexSearcher(gix).prepare(queries, RelevanceCollector(k, threshold))
    try:
        return b.stats()["work_items"]
    finally:
        b.close()


def assert_wide(gix, queries, k, threshold=INT_MAX):
    """The batch runs on bool_window_kernel: one work item per non-empty query and 1,048,576-doc slice."""
    want = n_nonempty(queries) * -(-gix.n_docs // WIDE_SLICE)
    got = work_items(gix, queries, k, threshold)
    assert got == want, f"expected a wide batch ({want} work items), got {got} work items"


def assert_probe(gix, queries, k, threshold=INT_MAX):
    """The batch runs on the probe kernel: at least one work item per non-empty query and 524,288-doc slice."""
    assert gix.n_docs > PROBE_SLICE
    n = n_nonempty(queries)
    got = work_items(gix, queries, k, threshold)
    assert got >= n * -(-gix.n_docs // PROBE_SLICE) > n * -(-gix.n_docs // WIDE_SLICE), f"expected a probe batch, got {got} items"


def oracle_pages(oix, queries, k, search_after=None):
    carr, ncl, qarr, nq = compile_queries(queries, search_after)
    return oracle.search_compiled(oix, carr, ncl, qarr, nq, k)


def as_tuple(res):
    return res.docs, res.scores, res.counts, res.total_hits, res.relation


def check_pages(res, want, threshold=INT_MAX, what=""):
    """assert_same_hits, plus the totalHits rule of both relations."""
    assert_same_hits(as_tuple(res), want, what=what)
    gte = res.relation != 0
    if threshold == INT_MAX:
        assert not gte.any(), f"{what}: COMPLETE mode reported GREATER_THAN_OR_EQUAL_TO"
    assert (res.total_hits[gte] > threshold).all() and (res.total_hits[gte] <= want[3][gte]).all(), f"{what}: lower-bound totalHits"


def same_pages(a, b, rows_a, rows_b, what=""):
    """Bit-identical pages of rows_a in a and rows_b in b (counts, docs, scores, totalHits, relation)."""
    for i, j in zip(rows_a, rows_b):
        n = int(a.counts[i])
        assert n == b.counts[j], f"{what} query {i}: counts {n} vs {b.counts[j]}"
        assert np.array_equal(a.docs[i, :n], b.docs[j, :n]), f"{what} query {i}: docs differ"
        assert np.array_equal(a.scores[i, :n].view(np.uint32), b.scores[j, :n].view(np.uint32)), f"{what} query {i}: scores differ"
        assert a.total_hits[i] == b.total_hits[j] and a.relation[i] == b.relation[j], f"{what} query {i}: totalHits differ"


_BYTE4 = np.array([oracle.int_to_byte4(n) for n in range(4096)], np.uint8)


def numpy_shard(n_docs, lists, seed=0, live_docs=None):
    """One text field with norms from numpy posting lists [(docs ascending, freqs)], one per term (ids in list order).
    A doc's length is the sum of its term frequencies plus 1..39 other tokens."""
    off = np.zeros(len(lists) + 1, np.int64)
    off[1:] = np.cumsum([len(d) for d, _ in lists])
    docs = np.concatenate([np.asarray(d, np.int32) for d, _ in lists])
    freqs = np.concatenate([np.asarray(f, np.int32) for _, f in lists])
    lengths = np.bincount(docs, weights=freqs, minlength=n_docs).astype(np.int64)
    lengths += np.random.default_rng(seed).integers(1, 40, n_docs)
    return ix.HostShard(n_docs=n_docs, doc_base=0, term_off=off, post_docs=docs, post_freqs=freqs,
                        fields=[ix.TextField(_BYTE4[lengths], n_docs, int(lengths.sum()))], live_docs=live_docs)


def disj(terms, boosts=None):
    q = BooleanQuery()
    for i, t in enumerate(terms):
        tq = TermQuery(int(t))
        q.add(BoostQuery(tq, boosts[i]) if boosts and boosts[i] != 1.0 else tq, Occur.SHOULD)
    return q


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(TermQuery(int(c)) if isinstance(c, (int, np.integer)) else c, o)
    return q


# ---------------------------------------------------------------- the 600K-doc corpus most tests share

def mix_shard():
    """600K synthetic docs (2 probe slices, 1 window slice); column 0 single-valued in [0, 1M), column 1 multi-valued
    (0..4 values in [-1000, 1000) per doc); appended terms: one without postings, and three with exactly 512, 513 and
    1024 postings spread over the shard. Returns (shard, {name: term id})."""
    sh = ix.synth_text_shard(N_MIX, 20_000, min_len=4, poisson_mean=12.0)
    rng = np.random.default_rng(17)
    cnt = rng.integers(0, 5, N_MIX)
    off = np.zeros(N_MIX + 1, np.int64)
    np.cumsum(cnt, out=off[1:])
    vals = rng.integers(-1000, 1000, int(off[-1])).astype(np.int64)
    vals = vals[np.lexsort((vals, np.repeat(np.arange(N_MIX), cnt)))]
    sh.columns = [ix.synth_int_column(N_MIX), vals]
    sh.column_has = [None, None]
    sh.column_offsets = [None, off]
    extra = {}
    docs, freqs, term_off = [sh.post_docs], [sh.post_freqs], list(sh.term_off)
    for name, df in (("empty", 0), ("k512", 512), ("k513", 513), ("k1024", 1024)):
        d = np.unique(np.linspace(0, N_MIX - 1, df).astype(np.int32)) if df else np.zeros(0, np.int32)
        assert len(d) == df
        docs.append(d)
        freqs.append((1 + (d % 4)).astype(np.int32))
        term_off.append(term_off[-1] + df)
        extra[name] = len(term_off) - 2
    sh.post_docs, sh.post_freqs = np.concatenate(docs), np.concatenate(freqs)
    sh.term_off = np.array(term_off, np.int64)
    return sh, extra


@pytest.fixture(scope="module")
def mix(gpu_ctx):
    sh, extra = mix_shard()
    gix = GpuIndex(gpu_ctx, sh)
    yield sh, oracle.OracleIndex(sh), gix, extra
    gix.close()


def mix_queries(extra, n=96, seed=41):
    """5-8 term clauses with every occur, minimum_number_should_match 0-3, clause and outer boosts, a repeated term, a
    term without postings, single- and multi-valued range clauses in every occur, match-all and range-led queries."""
    rng = np.random.default_rng(seed)
    qs = []
    for i in range(n):
        n_terms = 5 + i % 4
        pool = np.unique(np.floor(10 ** rng.uniform(0.3, 3.3, size=3 * n_terms)).astype(np.int64).clip(1, 19_999))
        ranks = sorted(int(r) for r in rng.choice(pool, size=min(n_terms, len(pool)), replace=False))
        while len(ranks) < n_terms:
            ranks.append(ranks[-1] + 1)
        if i % 7 == 0:
            ranks[-1] = ranks[1]                  # the same term twice
        if i % 6 == 1:
            ranks[-2] = extra["empty"]            # a term without postings
        q = BooleanQuery(minimum_number_should_match=(i // 2) % 4 if i % 3 else 0)
        pat = i % 8
        for j, r in enumerate(ranks):
            occ = Occur.SHOULD
            if j == 0 and pat in (1, 2, 3, 6):
                occ = Occur.MUST
            elif j == 1 and pat == 2:
                occ = Occur.FILTER
            elif j == 1 and pat == 3:
                occ = Occur.MUST
            elif j == 0 and pat == 4:
                occ = Occur.FILTER
            elif j == n_terms - 1 and pat in (3, 4, 5):
                occ = Occur.MUST_NOT
            tq = TermQuery(r)
            if (i + j) % 5 == 0:
                tq = BoostQuery(tq, (0.5, 2.0, 3.25)[j % 3])
            q.add(tq, occ)
        if i % 3 != 2:                            # a range clause; column alternates single / multi-valued
            r_occ = (Occur.FILTER, Occur.MUST, Occur.MUST_NOT, Occur.SHOULD)[(i // 3) % 4]
            if i % 2 == 0:
                lo = int(rng.integers(0, 700_000))
                rq = RangeQuery(0, lo, lo + 300_000)
            else:
                lo = int(rng.integers(-1100, 700))
                rq = RangeQuery(1, lo, lo + 600)
            q.add(BoostQuery(rq, 1.5) if i % 4 == 1 else rq, r_occ)
        if pat == 7:
            q.add(MatchAllDocsQuery(), Occur.MUST if i % 16 == 7 else Occur.SHOULD)   # no term can lead: dense sweep
        qs.append(BoostQuery(q, 1.75) if i % 5 == 2 else q)
    qs.append(bq(*[(r, Occur.SHOULD) for r in (1, 2, 3)], (4, Occur.MUST), (5, Occur.MUST), msm=4))   # matches nothing
    return qs


def test_clause_mix_5_to_8_terms(mix):
    """bool_window_kernel's pass 1 / 2 / 3 and evaluate_doc on 5-8 term clauses: MUST / FILTER / MUST_NOT / SHOULD, msm 0-3,
    boosts, a repeated term (two slots of one list), a term without postings, single- and multi-valued ranges in every
    occur, dense-driver sweeps. Catches a wrong driver choice (a required list that does not lead loses the docs it
    alone holds), a pass 2 / pass 3 that leaves a word set (phantom matches in the next window), a wrong slot mask for
    FILTER / MUST_NOT terms, a wrong score combination (ReqOptSumScorer float add vs ConjunctionScorer double add), or a
    multi-valued range evaluated as single-valued."""
    sh, oix, gix, extra = mix
    qs = mix_queries(extra)
    kinds = {type(c.query) for q in qs for c in (q.query if isinstance(q, BoostQuery) else q).clauses}
    assert {TermQuery, BoostQuery, RangeQuery, MatchAllDocsQuery} <= kinds
    assert n_nonempty(qs) < len(qs)   # msm above the SHOULD count: a query without work items rides along
    want = oracle_pages(oix, qs, 100)
    assert (want[2] == 100).any() and ((want[2] > 0) & (want[2] < 100)).any()
    s = GpuIndexSearcher(gix)
    for thr in (INT_MAX, 200):
        assert_wide(gix, qs, 100, thr)
        check_pages(s.search_batch(qs, RelevanceCollector(100, thr)), want, thr, what=f"clause mix thr={thr}")


def test_16_clauses_run_17_and_9_terms_refused(mix):
    """The clause limits of compile_batch: 8 term + 8 range clauses is the widest query the GPU path runs (and it runs
    wide, equal to the oracle); a 17th clause or a 9th term clause is UNSUPPORTED."""
    sh, oix, gix, extra = mix
    q16 = BooleanQuery()
    for r in (1, 3, 7, 20, 60, 150, 400, 900):
        q16.add(TermQuery(r), Occur.SHOULD)
    for j in range(8):
        if j == 6:
            q16.add(RangeQuery(1, 900, 999), Occur.MUST_NOT)
        else:
            q16.add(RangeQuery(0, 0, 900_000 - 50_000 * j), Occur.FILTER if j % 2 else Occur.SHOULD)
    assert_wide(gix, [q16], 50)
    check_pages(GpuIndexSearcher(gix).search_batch([q16], RelevanceCollector(50, INT_MAX)), oracle_pages(oix, [q16], 50), what="16 clauses")
    q17 = BooleanQuery(clauses=list(q16.clauses)).add(RangeQuery(1, 0, 10), Occur.FILTER)
    q9 = disj([1, 2, 3, 4, 5, 6, 7, 8, 9])
    s = GpuIndexSearcher(gix)
    for q, msg in ((q17, "more than 16 clauses"), (q9, "more than 8 term clauses")):
        with pytest.raises(NrtGpuUnsupported, match=msg):
            s.search_batch([q], RelevanceCollector(10, INT_MAX))


def test_wide_refusals(mix):
    """What the window engine cannot do is refused, never answered wrongly: sorted search and aggregations on a wide batch
    (5 term clauses, or top_k > 512), and top_k 1025 on any batch, are UNSUPPORTED."""
    sh, oix, gix, extra = mix
    s = GpuIndexSearcher(gix)
    wide5 = disj([1, 2, 3, 4, 5])
    narrow = disj([1, 2, 3])
    for q, k in ((wide5, 10), (narrow, 600)):
        with pytest.raises(NrtGpuUnsupported, match="sorted search"):
            s.search_sorted([q], SortFieldCollector(k, SortType(0)))
        with pytest.raises(NrtGpuUnsupported, match="aggregations"):
            s.search_with_collectors([q], RelevanceCollector(k, INT_MAX), [MinCollector(0)])
    with pytest.raises(NrtGpuUnsupported, match="top_k > 1024"):
        s.search_batch([narrow], RelevanceCollector(1025, INT_MAX))
    # the narrow shapes themselves are served (by the probe kernel)
    assert s.search_sorted([narrow], SortFieldCollector(10, SortType(0))).counts[0] == 10


def test_top_k_boundary_and_engine_agreement(mix):
    """The same 1-4-term queries at top_k 512 (probe kernel) and at 513 and 1024 (window kernel, 4096-key buffer and
    merge_slices_kernel at their largest top_k): every page equals the oracle, and the 512 / 513 pages are bit-identical
    prefixes of the 1024 page. Queries with exactly 512, 513 and 1024 matches and with fewer matches than k sit on every
    boundary. Catches an off-by-one in the keep / cut to top_k, a kth-key theta that drops the k-th hit, or a tie order
    that differs between the engines."""
    sh, oix, gix, extra = mix
    terms = ix.synth_query_terms(40, 4, 20_000, seed=901, log10_lo=0.3, log10_hi=3.5)
    qs = [disj(t[:1 + i % 4]) for i, t in enumerate(terms)]
    qs += [bq((int(terms[i][0]), Occur.MUST), (int(terms[i][1]), Occur.SHOULD)) for i in range(8)]
    qs += [TermQuery(extra["k512"]), disj([extra["k513"]]), TermQuery(extra["k1024"]),
           bq((extra["k1024"], Occur.MUST), (1, Occur.SHOULD)), disj([extra["k512"], extra["k513"]]),
           disj([15_000, 17_000]), TermQuery(19_000)]
    s = GpuIndexSearcher(gix)
    pages = {}
    for k in (512, 513, 1024):
        (assert_probe if k == 512 else assert_wide)(gix, qs, k)
        want = oracle_pages(oix, qs, k)
        pages[k] = s.search_batch(qs, RelevanceCollector(k, INT_MAX))
        check_pages(pages[k], want, what=f"top_k={k}")
    total = pages[1024].total_hits
    for v in (512, 513, 1024):
        assert (total == v).any(), f"no query with exactly {v} matches"
    assert (total < 512).any() and (total > 1024).any()
    full = pages[1024]
    for k in (512, 513):
        p = pages[k]
        assert np.array_equal(p.counts, np.minimum(full.counts, k)) and np.array_equal(p.total_hits, full.total_hits)
        for q in range(len(qs)):
            n = int(p.counts[q])
            assert np.array_equal(p.docs[q, :n], full.docs[q, :n]), f"top_k {k} query {q}: not a prefix of the 1024 page"
            assert np.array_equal(p.scores[q, :n].view(np.uint32), full.scores[q, :n].view(np.uint32))


def test_batch_composition_does_not_change_pages(mix):
    """One 6-term query appended to a batch of 3-term queries moves the whole batch from the probe kernel to the window
    kernel; the shared queries' pages must stay bit-identical (and equal to the oracle). Catches any engine difference a
    user would see only when an unrelated request shares the micro-batch."""
    sh, oix, gix, extra = mix
    terms = ix.synth_query_terms(64, 6, 20_000, seed=902, log10_lo=0.3, log10_hi=3.5)
    qs = [disj(t[:3]) if i % 3 else bq((int(t[0]), Occur.MUST), (int(t[1]), Occur.SHOULD), (int(t[2]), Occur.SHOULD))
          for i, t in enumerate(terms)]
    qs_wide = qs + [disj(terms[0])]
    assert_probe(gix, qs, 100)
    assert_wide(gix, qs_wide, 100)
    s = GpuIndexSearcher(gix)
    a = s.search_batch(qs, RelevanceCollector(100, INT_MAX))
    b = s.search_batch(qs_wide, RelevanceCollector(100, INT_MAX))
    check_pages(b, oracle_pages(oix, qs_wide, 100), what="with the 6-term query")
    same_pages(a, b, range(len(qs)), range(len(qs)), what="probe vs window batch")


def test_search_after_pages_of_600(mix):
    """searchAfter on the window kernel (top_k 600: `key < after_key` in offer, the after key of a doc past the shard):
    page 2 after the 600th hit equals the oracle's page 2, pages 1 + 2 are exactly the top-1024 page's first 1024 hits (no
    overlap, no gap), and totalHits is the same on both pages. Catches an after test that is inclusive (the 600th hit
    repeated) or that also drops equal-score docs after the after doc."""
    sh, oix, gix, extra = mix
    terms = ix.synth_query_terms(32, 6, 20_000, seed=903, log10_lo=0.3, log10_hi=3.2)
    qs = [disj(t[:2 + i % 5]) if i % 4 else bq((int(t[0]), Occur.MUST), *[(int(x), Occur.SHOULD) for x in t[1:5]])
          for i, t in enumerate(terms)]
    qs += [TermQuery(extra["k1024"]),                # exactly 1024 matches: pages 1 + 2 are the whole top-1024 page
           disj([extra["k512"], extra["k513"]])]     # a few under 1024: page 2 is short
    s = GpuIndexSearcher(gix)
    assert_wide(gix, qs, 600)
    p1 = s.search_batch(qs, RelevanceCollector(600, INT_MAX))
    check_pages(p1, oracle_pages(oix, qs, 600), what="page 1")
    sel = [q for q in range(len(qs)) if p1.counts[q] == 600]
    assert len(sel) > len(qs) // 2
    after = [ScoreDoc(int(p1.docs[q, 599]), float(p1.scores[q, 599])) for q in sel]
    sq = [qs[q] for q in sel]
    assert_wide(gix, sq, 600)
    p2 = s.search_batch(sq, RelevanceCollector(600, INT_MAX), search_after=after)
    check_pages(p2, oracle_pages(oix, sq, 600, after), what="page 2")
    full = s.search_batch(sq, RelevanceCollector(1024, INT_MAX))
    assert (p2.counts == 600).any() and (p2.counts == 424).any() and ((p2.counts > 0) & (p2.counts < 424)).any()
    for i, q in enumerate(sel):
        assert p1.total_hits[q] == p2.total_hits[i] == full.total_hits[i]
        docs = np.concatenate([p1.docs[q, :600], p2.docs[i, :p2.counts[i]]])[:1024]
        scores = np.concatenate([p1.scores[q, :600], p2.scores[i, :p2.counts[i]]])[:1024]
        n = int(full.counts[i])
        assert len(docs) == n and np.array_equal(docs, full.docs[i, :n]), f"query {q}: pages 1 + 2 differ from the top-1024 page"
        assert np.array_equal(scores.view(np.uint32), full.scores[i, :n].view(np.uint32))


def test_leaves_packed_merge_top_k_1024_search_after(gpu_ctx, mix):
    """GpuLeafSearcher over 3 leaves (doc_base 0, 150,000, 380,000) at top_k 1024 (the probe kernel takes top_k <= 512, so
    every leaf runs the window kernel): merge_pairs_kernel merges 3 x 1024 pairs, sums totalHits, and the whole-reader
    searchAfter doc lies in another leaf for most leaves (after_key: every doc of an earlier leaf follows it, every doc
    of a later leaf precedes it). Compared with the oracle on the whole reader. Catches a doc_base slip, a merge that keeps
    fewer than top_k pairs, or an after key that is wrong outside the after doc's own leaf."""
    sh, oix, gix, extra = mix
    cuts = (0, 150_000, 380_000, N_MIX)
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    assert [l.doc_base for l in leaves] == [0, 150_000, 380_000]
    terms = ix.synth_query_terms(24, 5, 20_000, seed=904, log10_lo=0.3, log10_hi=3.0)
    qs = [disj(t[:1 + i % 5]) if i % 3 else bq((int(t[0]), Occur.MUST), *[(int(x), Occur.SHOULD) for x in t[1:]])
          for i, t in enumerate(terms)]
    ls = GpuLeafSearcher(gpu_ctx, leaves)
    try:
        for l in leaves:
            assert_wide(l, qs, 1024)
        want = oracle_pages(oix, qs, 1024)
        check_pages(ls.search_batch(qs, RelevanceCollector(1024, INT_MAX)), want, what="3 leaves")
        sel = [q for q in range(len(qs)) if want[2][q] > 700]
        after = [ScoreDoc(int(want[0][q, 300 + 13 * i]), float(want[1][q, 300 + 13 * i])) for i, q in enumerate(sel)]
        leaf_of = np.searchsorted(cuts, [a.doc for a in after], side="right") - 1
        assert len(set(leaf_of.tolist())) >= 2, "the after docs should lie in different leaves"
        sq = [qs[q] for q in sel]
        got = ls.search_batch(sq, RelevanceCollector(1024, INT_MAX), search_after=after)
        check_pages(got, oracle_pages(oix, sq, 1024, after), what="3 leaves, searchAfter")
    finally:
        ls.close()
        for l in leaves:
            l.close()


# ---------------------------------------------------------------- numpy-built shards for the kernel's edges

def edge_shard():
    """n_docs = 1,048,576 + 3 * 16,384 + 77: two window slices, the second ending 77 docs into its fourth window.
    Terms 0-2 hold docs on both sides of every window edge (w * 16384 - 1, w * 16384), the slice edge (1,048,575 /
    1,048,576) and n_docs - 1 (term 1 with tf 255..300 on five of them); term 3 holds every doc of one window in each
    slice (16,384 candidates in one window, the first of slice 0 before any theta exists: compact_candidates runs
    mid-window) and every 97th doc elsewhere; term 4 straddles
    the slice edge; terms 5-16 hold 2 % of the docs each."""
    n = WIDE_SLICE + 3 * 16384 + 77
    m = np.arange(16384, n, 16384)
    edges = np.unique(np.concatenate([m - 1, m, [0, WIDE_SLICE - 1, WIDE_SLICE, n - 1]]))
    saturated = ((16383, 255), (16384 * 40, 256), (WIDE_SLICE - 1, 300), (WIDE_SLICE, 270), (n - 1, 260))
    e1 = np.unique(np.concatenate([edges[1::2], [d for d, _ in saturated]]))
    f1 = np.full(len(e1), 2, np.int32)
    for d, f in saturated:
        f1[np.searchsorted(e1, d)] = f
    e2 = edges[1::3]
    dense = np.unique(np.concatenate([np.arange(0, 16384), np.arange(WIDE_SLICE + 16384, WIDE_SLICE + 2 * 16384),
                                      np.arange(0, n, 97)]))
    straddle = np.arange(WIDE_SLICE - 5000, WIDE_SLICE + 5000)
    rng = np.random.default_rng(77)
    lists = [(edges, 1 + edges % 5), (e1, f1), (e2, np.ones(len(e2))), (dense, 1 + (dense * 7) % 11), (straddle, 1 + straddle % 3)]
    for _ in range(12):
        d = np.sort(rng.choice(n, n // 50, replace=False))
        lists.append((d, rng.integers(1, 4, len(d))))
    assert f1.max() >= 255
    return numpy_shard(n, lists, seed=78)


def test_window_and_slice_edges(gpu_ctx):
    """Window / slice arithmetic of bool_window_kernel at top_k 1024: the posting bounds at every window boundary
    (lower_bound at slice_base + w * 16384), the last partial window (wlen), the second slice's clamp to n_docs, the
    candidate buffer compacted in the middle of a window, exact_freq_slow at the edges. Catches an off-by-one in a window
    bound (the doc at w * 16384 - 1 lands in the wrong window and indexes slots[16384], or is lost), a slice end that
    drops n_docs - 1, or a mid-window compaction that loses a candidate or sets theta too high."""
    E0, E1, E2, D, Z = range(5)
    F = list(range(5, 17))
    sh = edge_shard()
    qs = [
        disj([E0, E1, E2, D, Z]),                                                # every list drives: ownership
        disj([D, F[0], F[1], F[2], F[3]]),                                       # dense window: compaction mid-window
        bq((D, Occur.MUST), (E0, Occur.SHOULD), (E1, Occur.SHOULD), (F[4], Occur.SHOULD), (F[5], Occur.SHOULD)),
        bq((E0, Occur.MUST), (D, Occur.SHOULD), (E1, Occur.SHOULD), (E2, Occur.SHOULD), (Z, Occur.SHOULD)),
        bq((D, Occur.SHOULD), (E0, Occur.SHOULD), (F[6], Occur.SHOULD), (F[7], Occur.SHOULD), (E2, Occur.MUST_NOT)),
        bq((E0, Occur.SHOULD), (E1, Occur.SHOULD), (E2, Occur.SHOULD), (D, Occur.SHOULD), (Z, Occur.SHOULD), msm=2),
        bq((Z, Occur.FILTER), (E0, Occur.SHOULD), (E1, Occur.SHOULD), (D, Occur.SHOULD), (F[8], Occur.SHOULD)),
        disj([F[9], F[10], F[11], E1, D], boosts=[1.0, 2.5, 1.0, 4.0, 0.5]),
        bq((F[0], Occur.MUST), (F[1], Occur.MUST), (E0, Occur.SHOULD), (D, Occur.SHOULD), (Z, Occur.SHOULD)),   # < k matches
        disj([E0, E1, E2, F[0], Z]),
        bq((MatchAllDocsQuery(), Occur.SHOULD), (E0, Occur.SHOULD), (E1, Occur.SHOULD), (D, Occur.SHOULD), (Z, Occur.SHOULD),
           (F[1], Occur.SHOULD)),                                                # dense driver over both slices
        bq((E1, Occur.MUST), (E0, Occur.SHOULD), (E2, Occur.SHOULD), (Z, Occur.SHOULD), (F[2], Occur.SHOULD)),   # tf >= 255 leads
    ]
    gix = GpuIndex(gpu_ctx, sh)
    try:
        assert_wide(gix, qs, 1024)
        want = oracle_pages(oracle.OracleIndex(sh), qs, 1024)
        check_pages(GpuIndexSearcher(gix).search_batch(qs, RelevanceCollector(1024, INT_MAX)), want, what="window / slice edges")
    finally:
        gix.close()
    assert (want[2] == 1024).sum() >= 6 and (want[2] < 1024).any()
    last = sh.n_docs - 1
    assert any(last in want[0][q, :want[2][q]] for q in range(len(qs))), "n_docs - 1 should be a hit of some page"


def test_ties_and_deletes_across_compactions_and_slices(gpu_ctx):
    """1.2M docs of a few distinct contents (thousands of docs per exact score), every 7th doc deleted, top_k 1024: ties
    resolve by doc ascending through every compact_candidates, the slice-wide theta (atomicMax of 64-bit keys) and
    merge_slices_kernel. The best-scoring group of one query is 1,500 identical docs straddling the slice edge at
    1,048,576, so the cut at 1024 falls inside one tie group that both slices hold. Catches a key whose doc part does
    not order equal scores by doc ascending, a cut to top_k (in a compaction or in the merge) that is not a total order
    on (score, doc), or deleted docs returned."""
    n = 1_200_000
    i = np.arange(n)
    w_lo, w_hi = WIDE_SLICE - 500, WIDE_SLICE + 1000
    in_w = (i >= w_lo) & (i < w_hi)
    X, Y, Zt, U, V, W = range(6)
    sel = [np.ones(n, bool), (i % 3 != 0) & ~in_w, (i % 3 == 0) & ~in_w, (i % 5 == 0) & ~in_w, (i % 11 == 0) & ~in_w, in_w]
    tf = [1, 2, 1, 1, 1, 3]
    lists = [(i[s], np.full(int(s.sum()), f)) for s, f in zip(sel, tf)]
    live = np.ones(n, np.uint8)
    live[::7] = 0
    sh = numpy_shard(n, lists, live_docs=live)
    length = 2 + sum(f * s for s, f in zip(sel, tf))
    sh.fields[0] = ix.TextField(_BYTE4[length], n, int(length.sum()))   # identical content -> identical norms
    qs = [disj([X, Y, Zt, U, V]),
          disj([W, X, Y, U, V]),
          bq((X, Occur.MUST), (Y, Occur.SHOULD), (Zt, Occur.SHOULD), (U, Occur.SHOULD), (V, Occur.SHOULD)),
          bq((X, Occur.FILTER), (Y, Occur.SHOULD), (Zt, Occur.SHOULD), (U, Occur.SHOULD), (V, Occur.SHOULD)),
          bq((X, Occur.SHOULD), (Y, Occur.SHOULD), (U, Occur.SHOULD), (V, Occur.SHOULD), (Zt, Occur.MUST_NOT))]
    gix = GpuIndex(gpu_ctx, sh)
    try:
        assert_wide(gix, qs, 1024)
        want = oracle_pages(oracle.OracleIndex(sh), qs, 1024)
        got = GpuIndexSearcher(gix).search_batch(qs, RelevanceCollector(1024, INT_MAX))
    finally:
        gix.close()
    check_pages(got, want, what="ties + deletes")
    for q in range(len(qs)):
        assert got.counts[q] == 1024 and got.scores[q, 0] == got.scores[q, 1023], f"query {q}: the page should be one tie group"
        assert (np.diff(got.docs[q]) > 0).all() and live[got.docs[q]].all()
    d = got.docs[1]
    assert (d < WIDE_SLICE).any() and (d >= WIDE_SLICE).any(), "the tie group should span both slices"


def test_tf_saturation_omit_norms_two_fields(gpu_ctx):
    """exact_freq_slow on the window path: the 3,000-doc two-field corpus of the parity suite (body with norms and docs
    of tf 300..600, title with omitNorms) under 5-term queries, at top_k 100 and 1024. The shard is one window slice of
    either engine, so the item count cannot tell them apart: the routing rule alone (5 term clauses) puts the batch on
    the window kernel. Catches a saturated byte scored as tf 255, an exception looked up at the wrong posting, or the
    norms of one field read for the other."""
    rng = np.random.default_rng(3)
    body, title = [], []
    for d in range(3000):
        n = int(rng.integers(3, 60))
        toks = [f"w{int(x)}" for x in rng.zipf(1.3, n) if x < 200]
        if d % 500 == 0:
            toks += ["w1"] * (300 + d // 10)
        body.append(toks or ["w1"])
        title.append([f"w{int(x)}" for x in rng.zipf(1.5, 4) if x < 50] if d % 3 else [])
    sh, vocab = shard_from_token_docs([body, title], omit_norms=[False, True])
    assert sh.post_freqs.max() >= 255
    b = lambda w: vocab[(0, w)]
    t = lambda w: vocab[(1, w)]
    qs = [disj([b("w1"), t("w1"), b("w2"), t("w2"), b("w3")]),
          bq((b("w1"), Occur.MUST), (t("w2"), Occur.SHOULD), (b("w4"), Occur.SHOULD), (t("w3"), Occur.SHOULD), (b("w5"), Occur.SHOULD)),
          bq((t("w1"), Occur.MUST), (b("w3"), Occur.MUST), (b("w1"), Occur.SHOULD), (t("w4"), Occur.SHOULD), (b("w2"), Occur.SHOULD)),
          bq((b("w1"), Occur.FILTER), (b("w1"), Occur.SHOULD), (t("w1"), Occur.SHOULD), (b("w6"), Occur.SHOULD), (t("w5"), Occur.SHOULD)),
          bq((b("w1"), Occur.SHOULD), (b("w2"), Occur.SHOULD), (b("w3"), Occur.SHOULD), (t("w1"), Occur.SHOULD), (t("w2"), Occur.SHOULD), msm=2),
          BoostQuery(disj([b("w1"), b("w7"), t("w6"), b("w8"), t("w1")], boosts=[2.0, 1.0, 0.75, 1.0, 3.0]), 1.5)]
    oix = oracle.OracleIndex(sh)
    gix = GpuIndex(gpu_ctx, sh)
    try:
        s = GpuIndexSearcher(gix)
        for k in (100, 1024):
            assert_wide(gix, qs, k)
            check_pages(s.search_batch(qs, RelevanceCollector(k, INT_MAX)), oracle_pages(oix, qs, k), what=f"tf >= 255, top_k={k}")
    finally:
        gix.close()


# ---------------------------------------------------------------- limits: deadline and terminateAfter on wide batches

EXPIRED = dict(timeout_sec=0.5, elapsed_sec=1.0)   # the request's budget was spent before the call


def limit_queries():
    """48 wide queries (5-6 term clauses) and 48 probe queries (3 term clauses), none of them empty."""
    terms = ix.synth_query_terms(48, 6, 20_000, seed=906, log10_lo=0.3, log10_hi=3.8)
    wide = [disj(t[:5 + i % 2]) if i % 2 else bq((int(t[0]), Occur.MUST), *[(int(x), Occur.SHOULD) for x in t[1:5]])
            for i, t in enumerate(terms)]
    narrow = [disj(t[:3]) for t in terms]
    return wide, narrow


def test_wide_terminate_after_contract(mix):
    """terminateAfter on the window kernel (flagged by merge_slices_kernel from the counted hits, capped at
    terminateAfterMaxRecallCount by the fetch): the contract of test_gpu_limits.py::test_terminate_after_contract --
    terminatedEarly iff more than terminateAfter docs match, totalHits in [terminateAfter, min(matches, maxRecall)] with
    GREATER_THAN_OR_EQUAL_TO, every hit a true match with its exact score, untouched queries equal to the unlimited
    search. Catches the flag or the recall cap not applied on this engine."""
    sh, oix, gix, extra = mix
    qs, _ = limit_queries()
    k = 50
    assert_wide(gix, qs, k)
    carr, ncl, qarr, nq = compile_queries(qs)
    want = oracle.search_compiled(oix, carr, ncl, qarr, nq, k)
    matches = want[3]
    T = int(np.median(matches))
    R = 2 * T
    assert T > 0
    s = GpuIndexSearcher(gix)
    res = s.search_batch(qs, RelevanceCollector(k, INT_MAX, terminate_after=T, terminate_after_max_recall_count=R))
    full = s.search_batch(qs, RelevanceCollector(k, INT_MAX))
    od, os_, oc, ot, orel, oterm = oracle.search_terminate_after(oix, carr, ncl, qarr, nq, k, T, R)
    assert np.array_equal(res.terminated_early, oterm)
    assert np.array_equal(oterm != 0, matches > T)
    t = res.terminated_early != 0
    assert t.any() and (~t).any()
    assert (res.relation[t] == 1).all() and not res.hit_timeout.any()
    assert (res.total_hits[t] >= T).all() and (res.total_hits[t] <= np.minimum(matches[t], R)).all()
    check_pages(full, want, what="unlimited")
    u = np.nonzero(~t)[0]
    same_pages(res, full, u, u, what="not terminated vs unlimited")
    for q in u:   # ... and the oracle under the wrapper
        n = int(oc[q])
        assert res.counts[q] == n and np.array_equal(res.docs[q, :n], od[q, :n]) and res.total_hits[q] == matches[q]
    sel =[int(q) for q in np.nonzero(t)[0][:12]]
    carr2, ncl2, qarr2, nq2 = compile_queries([qs[q] for q in sel])
    deep = 4096
    dd, ds, dc, _, _ = oracle.search_compiled(oix, carr2, ncl2, qarr2, nq2, deep)
    for i, q in enumerate(sel):
        truth = {int(d): s_ for d, s_ in zip(dd[i, :dc[i]], ds[i, :dc[i]])}
        for d, sc in zip(res.docs[q, :res.counts[q]], res.scores[q, :res.counts[q]]):
            if int(d) in truth:
                assert np.float32(sc).view(np.uint32) == np.float32(truth[int(d)]).view(np.uint32)
            else:
                assert dc[i] == deep and sc <= ds[i, deep - 1]


def test_wide_deadline(mix):
    """The deadline on the window kernel (deadline_passed at each work item's start): a generous deadline changes
    nothing; an expired one skips every work item -- hitTimeout on every query, GREATER_THAN_OR_EQUAL_TO, no hits, no
    count -- or raises CollectionTimeoutException with disallowPartialResults; a deadline that falls inside a large batch
    returns, per query, either the full page or a flagged partial one. Catches a window kernel that ignores the deadline
    (full results reported as on time)."""
    sh, oix, gix, extra = mix
    qs, _ = limit_queries()
    k = 20
    assert_wide(gix, qs, k)
    s = GpuIndexSearcher(gix)
    full = s.search_batch(qs, RelevanceCollector(k, INT_MAX))
    check_pages(full, oracle_pages(oix, qs, k), what="unlimited")
    ok = s.search_batch(qs, RelevanceCollector(k, INT_MAX, timeout_sec=120.0))
    assert not ok.hit_timeout.any()
    same_pages(ok, full, range(len(qs)), range(len(qs)), what="generous deadline")
    late = s.search_batch(qs, RelevanceCollector(k, INT_MAX, **EXPIRED))
    assert late.hit_timeout.all(), f"{int((late.hit_timeout == 0).sum())} of {len(qs)} queries ran past an expired deadline"
    assert (late.relation == 1).all() and (late.counts == 0).all() and (late.total_hits == 0).all()
    with pytest.raises(CollectionTimeoutException, match="Search collection exceeded timeout of"):
        s.search_batch(qs, RelevanceCollector(k, INT_MAX, disallow_partial_results=True, **EXPIRED))
    mid = s.search_batch(qs * 8, RelevanceCollector(k, INT_MAX, timeout_sec=20e-6))
    to = mid.hit_timeout != 0
    assert (mid.relation[to] == 1).all() and (mid.total_hits <= np.tile(full.total_hits, 8)).all()
    on_time = np.nonzero(~to)[0]
    same_pages(mid, full, on_time, on_time % len(qs), what="deadline inside the batch, queries on time")


def test_timeout_flags_do_not_leak_between_calls(mix):
    """Workspaces are pooled per index, so a call reads the timed_out flags its own run wrote only if the run clears them
    first, whatever engine it uses. An expired probe call followed by a wide call with a 120 s deadline (same nq, same
    pooled workspace), and an expired wide call followed by a probe call: the second call reports no hitTimeout, does not
    raise under disallowPartialResults, and returns the unlimited pages. Catches the flags cleared only on the probe
    kernel's launch path."""
    sh, oix, gix, extra = mix
    wide, narrow = limit_queries()
    k = 20
    assert len(wide) == len(narrow)
    assert_wide(gix, wide, k)
    assert_probe(gix, narrow, k)
    s = GpuIndexSearcher(gix)
    full = {id(wide): s.search_batch(wide, RelevanceCollector(k, INT_MAX)),
            id(narrow): s.search_batch(narrow, RelevanceCollector(k, INT_MAX))}
    for first, second, what in ((narrow, wide, "probe then wide"), (wide, narrow, "wide then probe")):
        assert s.search_batch(first, RelevanceCollector(k, INT_MAX, **EXPIRED)).hit_timeout.all()
        r = s.search_batch(second, RelevanceCollector(k, INT_MAX, timeout_sec=120.0))
        assert not r.hit_timeout.any(), f"{what}: {int(r.hit_timeout.sum())} queries report a timeout of the previous call"
        assert not r.relation.any()
        same_pages(r, full[id(second)], range(len(second)), range(len(second)), what=what)
        assert s.search_batch(first, RelevanceCollector(k, INT_MAX, **EXPIRED)).hit_timeout.all()
        r = s.search_batch(second, RelevanceCollector(k, INT_MAX, timeout_sec=120.0, disallow_partial_results=True))
        same_pages(r, full[id(second)], range(len(second)), range(len(second)), what=f"{what}, disallowPartialResults")


def test_empty_batch_after_expired_call(mix):
    """A batch with no work items at all (every query matches nothing) launches no search kernel; with a generous deadline
    after an expired call on the same index it must still report no timeout. Catches flags cleared only inside the
    `n_work > 0` branch."""
    sh, oix, gix, extra = mix
    wide, narrow = limit_queries()
    k = 20
    empty = [BooleanQuery(minimum_number_should_match=2).add(TermQuery(1), Occur.SHOULD) if i % 2 else BooleanQuery()
             for i in range(len(narrow))]
    assert work_items(gix, empty, k) == 0
    s = GpuIndexSearcher(gix)
    for first in (narrow, wide):
        assert s.search_batch(first, RelevanceCollector(k, INT_MAX, **EXPIRED)).hit_timeout.all()
        r = s.search_batch(empty, RelevanceCollector(k, INT_MAX, timeout_sec=120.0, disallow_partial_results=True))
        assert not r.hit_timeout.any() and not r.relation.any()
        assert not r.counts.any() and not r.total_hits.any()


# ---------------------------------------------------------------- a 2.3M-doc shard: three window slices

def test_multi_slice_top_k_1024(gpu_ctx):
    """2.3M docs (3 window slices), 64 queries of 5-6 terms at top_k 1024: merge_slices_kernel merges 3 x 1024 keys per
    query (the flat prefix scan over the non-empty lists, the cut to top_k), totalHits summed over the slices. Catches a
    merge that reads a list at the wrong offset, keeps one list too few, or drops keys when the buffer is full."""
    sh = ix.synth_text_shard(2_300_000, 50_000, min_len=4, poisson_mean=12.0)
    terms = ix.synth_query_terms(64, 6, 50_000, seed=905, log10_lo=0.3, log10_hi=3.0)
    qs = [disj(t[:5 + i % 2]) if i % 4 else bq((int(t[0]), Occur.MUST), *[(int(x), Occur.SHOULD) for x in t[1:]])
          for i, t in enumerate(terms)]
    gix = GpuIndex(gpu_ctx, sh)
    try:
        assert_wide(gix, qs, 1024)
        got = GpuIndexSearcher(gix).search_batch(qs, RelevanceCollector(1024, INT_MAX))
    finally:
        gix.close()
    want = oracle_pages(oracle.OracleIndex(sh), qs, 1024)
    check_pages(got, want, what="3 slices, top_k 1024")
    assert (want[2] == 1024).sum() >= 48
