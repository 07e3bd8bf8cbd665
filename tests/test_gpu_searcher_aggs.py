"""Aggregations over the leaves of a searcher (nrtgpu_searcher_search_bool_aggs_nested, GpuLeafSearcher.search_with_collectors):
terms buckets counted by value across leaves through the searcher's reader-wide dictionaries, min / max / sum, nested
collectors and nested top hits chosen per reader-wide bucket over every leaf.

The shard is the 1.1M-doc shard of tests/test_gpu_aggregations.py and tests/test_gpu_nested_aggs.py (doc_base 1000, every
11th doc deleted), cut into uneven doc-range leaves: one cut inside a probe slice, one leaf of a few dozen docs. Columns
added here make the union of the leaves' dictionaries matter: values in disjoint ranges per leaf, values in one leaf only
(the others hold none), 2049 distinct values reader-wide but at most 1025 in any leaf (the 2048-bucket chunk of the
selection is crossed only reader-wide), and two values whose counts tie only when summed over the leaves. Every result is
checked against the whole shard's references and against the single-image search of the whole shard: hits, score bits,
totalHits, keys, counts, n / totalBuckets / otherCounts, MIN / MAX and top hits exactly, SUM within n * 2^-53 * sum|v|."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import oracle
import test_gpu_aggregations as ta
import test_gpu_nested_aggs as tn
from helpers import shard_from_token_docs
from nrtsearch_b200 import NrtGpuError, NrtGpuUnsupported, _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, GpuIndex, GpuIndexSearcher, GpuLeafSearcher, MatchAllDocsQuery, MaxCollector,
                                   MinCollector, Occur, RangeQuery, RelevanceCollector, SumCollector, TermQuery, TermsCollector,
                                   TopHitsCollector, compile_queries)
from test_gpu_aggregations import C_INT, F64, MV, N, QUERIES, UNIQ, VOCAB, make_columns

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
K = 50
DOC_BASE = 1000
# leaf boundaries: a cut inside the first probe slice, a leaf of 37 docs, two large leaves
CUTS = [0, 300_001, 300_038, 750_000, N]
# columns added to make_columns' 13
DISJ, ONE_LEAF, WIDE, TIE = MV + 1, MV + 2, MV + 3, MV + 4
ONE_LEAF_AT = 2                     # the leaf that holds ONE_LEAF's values
WIDE_START = [0, 500, 700, 1024]    # leaf l holds WIDE keys [start, start + 1025): 2049 reader-wide
TIE_A, TIE_B = -5, 7                # 400 live docs each over leaves 0 and 3, 300 / 100 in one and 100 / 300 in the other


def added_columns(live):
    """DISJ, ONE_LEAF, WIDE, TIE over the whole shard (live: the whole shard's live docs)"""
    doc = np.arange(N, dtype=np.int64)
    leaf = np.searchsorted(CUTS, doc, side="right") - 1
    disj = leaf * 1_000_000 + doc % 37
    one = doc % 11 + 100
    one_has = (leaf == ONE_LEAF_AT).astype(np.uint8)
    keys = np.sort(np.random.default_rng(0xA6A).choice(np.arange(-2**40, 2**40, 2**20 + 7, dtype=np.int64), 2049, replace=False))
    wide = keys[np.asarray(WIDE_START)[leaf] + (doc - np.asarray(CUTS)[leaf]) % 1025]
    tie = np.zeros(N, np.int64)
    tie_has = np.zeros(N, np.uint8)
    for l, (na, nb) in ((0, (300, 100)), (3, (100, 300))):
        d = doc[(leaf == l) & (live != 0)][: na + nb]
        tie[d[:na]], tie[d[na:]] = TIE_A, TIE_B
        tie_has[d] = 1
    return [disj, one, wide, tie], [None, one_has, None, tie_has]


def whole_shard():
    sh = ix.synth_text_shard(N, VOCAB, seed=0xA66, min_len=4, poisson_mean=10.0)
    sh.columns, sh.column_has, offs = make_columns(N, 0xA67)
    sh.live_docs = (np.arange(N) % 11 != 0).astype(np.uint8)
    cols, has = added_columns(sh.live_docs)
    sh.columns += cols
    sh.column_has += has
    sh.column_offsets = [None] * MV + [offs] + [None] * len(cols)
    sh.doc_base = DOC_BASE
    return sh


@pytest.fixture(scope="module")
def shard(gpu_ctx):
    sh = whole_shard()
    whole = GpuIndex(gpu_ctx, sh)
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(lo, hi)) for lo, hi in zip(CUTS, CUTS[1:])]
    searcher = GpuLeafSearcher(gpu_ctx, leaves)
    oix = oracle.OracleIndex(sh)
    yield sh, whole, leaves, searcher, oix
    searcher.close()
    for g in leaves + [whole]:
        g.close()


@pytest.fixture(scope="module")
def ref(shard):
    sh, _, _, _, oix = shard
    return ta.Reference(sh, oix, QUERIES)


@pytest.fixture(scope="module")
def nref(shard):
    sh, _, _, _, oix = shard
    return tn.Ref(sh, oix, QUERIES)


def terms(c, size, desc=True, nested=(), order_by=None):
    return TermsCollector(c, size, desc, ta.FIELD_TYPE.get(c, "long"), tuple(nested), order_by)


# terms over the added columns, 8 per search: disjoint leaf ranges, one leaf only, 2049 values, a tie across leaves
ADDED = [terms(DISJ, 7), terms(DISJ, 2048, False), terms(ONE_LEAF, 5), terms(WIDE, 2048), terms(WIDE, 2047, False),
         terms(TIE, 1), terms(TIE, 2, False), terms(WIDE, 3)]
ADDED_NESTED = [
    terms(WIDE, 2048, nested=[("max", MaxCollector(DISJ, "long")), ("hits", TopHitsCollector(3))]),
    terms(TIE, 2, nested=[("hits", TopHitsCollector(5, 1)), ("sum", SumCollector(C_INT, "int"))]),
    terms(DISJ, 5, nested=[("min", MinCollector(WIDE, "long"))], order_by="min"),
    terms(ONE_LEAF, 4, False, nested=[("hits", TopHitsCollector(2))]),
]


def assert_same_hits(a, b):
    """the same pages (a single-image page leaves the slots past a query's count unset) and totalHits"""
    assert np.array_equal(a.counts, b.counts) and np.array_equal(a.total_hits, b.total_hits)
    for q, c in enumerate(a.counts.tolist()):
        assert np.array_equal(a.docs[q, :c], b.docs[q, :c]), f"query {q}: docs"
        assert np.array_equal(a.scores[q, :c].view(np.uint32), b.scores[q, :c].view(np.uint32)), f"query {q}: scores"


def assert_same_aggs(adds, x, y):
    """everything but the sums, whose atomics add in no fixed order"""
    for a, o, p in zip(adds, x, y):
        if not isinstance(a, TermsCollector):
            if not isinstance(a, SumCollector):
                assert np.array_equal(o.view(np.uint64), p.view(np.uint64)), type(a).__name__
            continue
        for f in ("keys", "counts", "n", "total_buckets", "other_counts"):
            assert np.array_equal(o[f], p[f]), f"terms column {a.column} size {a.size}: {f}"
        for name, c in a.nested:
            g, h = o["nested"][name], p["nested"][name]
            if isinstance(c, TopHitsCollector):
                assert all(np.array_equal(g[f], h[f]) for f in ("docs", "counts", "total_hits")), name
                assert np.array_equal(g["scores"].view(np.uint32), h["scores"].view(np.uint32)), name
            elif not isinstance(c, SumCollector):
                assert np.array_equal(g.view(np.uint64), h.view(np.uint64)), name


def search_both(shard, queries, adds, k=K):
    """(searcher result, single-image result of the whole shard); the hits and everything but sums agree"""
    _, whole, _, searcher, _ = shard
    got = searcher.search_with_collectors(queries, RelevanceCollector(k, INT_MAX), adds)
    one = GpuIndexSearcher(whole).search_with_collectors(queries, RelevanceCollector(k, INT_MAX), adds)
    assert_same_hits(got[0], one[0])
    assert_same_aggs(adds, got[1], one[1])
    return got


def test_leaves_make_the_union_matter(shard):
    sh = shard[0]

    def distinct(c, lo, hi):
        h = sh.column_has[c]
        return len(np.unique(sh.columns[c][lo:hi] if h is None else sh.columns[c][lo:hi][h[lo:hi] != 0]))

    spans = list(zip(CUTS, CUTS[1:]))
    assert [distinct(ONE_LEAF, lo, hi) for lo, hi in spans] == [0, 0, 11, 0]
    assert max(distinct(WIDE, lo, hi) for lo, hi in spans) == 1025 and distinct(WIDE, 0, N) == 2049
    assert distinct(DISJ, 0, N) == sum(distinct(DISJ, lo, hi) for lo, hi in spans)
    live = (sh.live_docs != 0) & (sh.column_has[TIE] != 0)
    assert (sh.columns[TIE][live] == TIE_A).sum() == (sh.columns[TIE][live] == TIE_B).sum() == 400
    for lo, hi in spans:
        assert (sh.columns[TIE][lo:hi][live[lo:hi]] == TIE_A).sum() != (sh.columns[TIE][lo:hi][live[lo:hi]] == TIE_B).sum() or \
            not live[lo:hi].any()


@pytest.mark.parametrize("group", range(len(ta.GROUPS) + 1))
def test_aggregations_match_whole_shard(shard, ref, group):
    adds = ta.GROUPS[group] if group < len(ta.GROUPS) else ADDED
    res, outs = search_both(shard, QUERIES, adds)
    ta.check_aggs(ref, adds, outs)
    assert res.total_hits.tolist() == [int(m.sum()) for m in ref.match]


@pytest.mark.parametrize("group", range(len(tn.GROUPS) + 1))
def test_nested_match_whole_shard(shard, nref, group):
    adds = tn.GROUPS[group] if group < len(tn.GROUPS) else ADDED_NESTED
    _, outs = search_both(shard, QUERIES, adds)
    for a, o in zip(adds, outs):
        if isinstance(a, TermsCollector):
            tn.check_terms(nref, a, o)


def test_tie_only_summed_over_leaves(shard):
    _, outs = search_both(shard, [MatchAllDocsQuery()], [terms(TIE, 1), terms(TIE, 2)])
    assert outs[0]["keys"][0].tolist() == [TIE_A] and outs[0]["counts"][0].tolist() == [400]
    assert outs[0]["other_counts"][0] == 400 and outs[0]["total_buckets"][0] == 2
    assert outs[1]["keys"][0].tolist() == [TIE_A, TIE_B] and outs[1]["counts"][0].tolist() == [400, 400]


def test_known_answers(gpu_ctx):
    """NestedCollectorOrderTest / NestedCollectionTest on the 100-doc shard cut into three leaves; the top hits of a
    MatchAllDocsQuery all score 1.0, so the global doc decides across the cut at doc 5"""
    i, j = np.repeat(np.arange(1, 6), 20), np.tile(np.arange(1, 21), 5)
    docs = [["a"] * (1 + d // 10) + ["b"] * (9 - d // 10) for d in range(100)]
    ids = np.arange(100, dtype=np.int64)
    sh, vocab = shard_from_token_docs([docs], columns=[i.astype(np.int64), (i * j).astype(np.int64), (-i * j).astype(np.int64),
                                                       ids % 2])
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(lo, hi)) for lo, hi in ((0, 5), (5, 61), (61, 100))]
    s = GpuLeafSearcher(gpu_ctx, leaves)
    try:
        for desc, keys in ((True, [1, 2, 3, 4, 5]), (False, [5, 4, 3, 2, 1])):
            for size, other in ((5, 0), (2, 60), (10, 0)):
                a = TermsCollector(0, size, desc, "int", (("max_order", MaxCollector(2, "int")), ("additional", MaxCollector(1, "int"))),
                                   "max_order")
                _, outs = s.search_with_collectors([MatchAllDocsQuery(), RangeQuery(0, 2, 4)], RelevanceCollector(10), [a])
                o, n = outs[0], min(size, 5)
                assert o["n"][0] == n and o["total_buckets"][0] == 5 and o["other_counts"][0] == other
                assert o["keys"][0, :n].tolist() == keys[:n]
                assert o["nested"]["max_order"][0, :n].tolist() == [-float(k) for k in keys[:n]]
                assert o["nested"]["additional"][0, :n].tolist() == [20.0 * k for k in keys[:n]]
                rk = [k for k in keys if 2 <= k <= 4][:size]
                assert o["keys"][1, :len(rk)].tolist() == rk and o["total_buckets"][1] == 3
                assert o["other_counts"][1] == 20 * (3 - len(rk))
        a = TermsCollector(3, 2, True, "int", (("nested", TopHitsCollector(5)),))
        res, outs = s.search_with_collectors([TermQuery(vocab[(0, "a")])], RelevanceCollector(10), [a])
        o = outs[0]
        assert sorted(o["keys"][0].tolist()) == [0, 1] and o["counts"][0].tolist() == [50, 50]
        h = o["nested"]["nested"]
        for b, key in enumerate(o["keys"][0].tolist()):
            assert h["total_hits"][0, b] == 50 and h["counts"][0, b] == 5
            assert h["docs"][0, b].tolist() == [90 + key, 92 + key, 94 + key, 96 + key, 98 + key]
            assert h["scores"][0, b].view(np.uint32).tolist() == [res.scores[0, 0].view(np.uint32)] * 5
        tn.check_terms(tn.Ref(sh, oracle.OracleIndex(sh), [TermQuery(vocab[(0, "a")])]), a, o)
        _, outs = s.search_with_collectors([MatchAllDocsQuery()], RelevanceCollector(10), [a])
        h = outs[0]["nested"]["nested"]
        for b, key in enumerate(outs[0]["keys"][0].tolist()):
            assert h["docs"][0, b].tolist() == [key, 2 + key, 4 + key, 6 + key, 8 + key]
            assert h["scores"][0, b].tolist() == [1.0] * 5
    finally:
        s.close()
        for g in leaves:
            g.close()


def test_top_hits_in_query_groups(shard, nref):
    """80 queries whose returned buckets hold every live doc: more than one pass-2 group of 2^26 keys over the leaves"""
    sh, _, _, _, oix = shard
    qs = [RangeQuery(C_INT, -30, 30)] * 80
    a = terms(C_INT, 60, nested=[("hits", TopHitsCollector(5)), ("max", MaxCollector(F64, "double"))])
    res, outs = search_both(shard, qs, [a], k=10)
    assert res.total_hits[0] * 80 > 2**26
    tn.check_terms(tn.Ref(sh, oix, qs[:1]), a, outs[0], rows=[0])


def test_one_leaf_is_the_single_image(shard, nref):
    """exactly the single image's results, but for the sums, held to the reference's bound"""
    _, whole, _, _, _ = shard
    s = GpuLeafSearcher(whole.ctx, [whole])
    try:
        for adds in (tn.GROUPS[0], ta.GROUPS[0]):
            got = s.search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX), adds)
            one = GpuIndexSearcher(whole).search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX), adds)
            assert_same_hits(got[0], one[0])
            assert_same_aggs(adds, got[1], one[1])
            for a, o in zip(adds, got[1]):
                if isinstance(a, TermsCollector) and a.nested:
                    tn.check_terms(nref, a, o)
    finally:
        s.close()


def test_repeated_call_is_identical(shard):
    """the second call reads the cached dictionaries"""
    _, _, _, searcher, _ = shard
    adds = tn.GROUPS[0] + [terms(WIDE, 2048)]
    r1, o1 = searcher.search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX), adds)
    r2, o2 = searcher.search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX), adds)
    assert_same_hits(r1, r2)
    assert_same_aggs(adds, o1, o2)


class _Restricted(ta.Reference):
    """a Reference of a doc-range prefix of a shard: the whole shard's match sets cut to the prefix"""

    def __init__(self, sh, match):
        self.sh, self.match, self._codes = sh, match, {}


def test_deletes_and_new_reader_versions(shard, gpu_ctx):
    sh, _, leaves, searcher, _ = shard
    adds = [terms(C_INT, 7), terms(DISJ, 2048), terms(WIDE, 2048), terms(TIE, 2), ta.stat(MinCollector, ta.I64),
            ta.stat(MaxCollector, F64), ta.stat(SumCollector, C_INT)]
    qs = QUERIES[:13]
    # more deletes in leaf 2 only
    lo, hi = CUTS[2], CUTS[3]
    live = sh.live_docs.copy()
    live[lo:hi] &= (np.arange(lo, hi) % 7 != 3).astype(np.uint8)
    try:
        leaves[2].set_live_docs(live[lo:hi])
        sh2 = dataclasses.replace(sh, live_docs=live)
        _, outs = searcher.search_with_collectors(qs, RelevanceCollector(K, INT_MAX), adds)
        ta.check_aggs(ta.Reference(sh2, oracle.OracleIndex(sh2), qs), adds, outs)
    finally:
        leaves[2].set_live_docs(sh.live_docs[lo:hi])
    # reader version 1: the first three leaves; version 2: the same images and a new leaf holding new values
    ref = ta.Reference(sh, oracle.OracleIndex(sh), qs)
    v1 = GpuLeafSearcher(gpu_ctx, leaves[:3])
    try:
        _, outs = v1.search_with_collectors(qs, RelevanceCollector(K, INT_MAX), adds[:4])
        cut = CUTS[3]
        prefix = sh.doc_range(0, cut, doc_base=DOC_BASE)
        ta.check_aggs(_Restricted(prefix, [m[:cut] for m in ref.match]), adds[:4], outs)
    finally:
        v1.close()
    v2 = GpuLeafSearcher(gpu_ctx, leaves)
    try:
        _, outs = v2.search_with_collectors(qs, RelevanceCollector(K, INT_MAX), adds)
        ta.check_aggs(ref, adds, outs)
    finally:
        v2.close()


def raw(searcher, queries, aggs, nested, k=K):
    """nrtgpu_searcher_search_bool_aggs_nested with hand-made records; returns the output buffers"""
    lib = _native.gpu_lib()
    carr, ncl, qarr, nq = compile_queries(queries)
    arr = (_native.Aggregation * max(len(aggs), 1))(*aggs)
    bufs = [np.zeros(nq * max(a.size, 1), np.int64) for a in aggs]
    res = (_native.AggregationResult * max(len(aggs), 1))(*[_native.AggregationResult(b.ctypes.data, b.ctypes.data, None, None, None, None)
                                                            for b in bufs])
    narr = (_native.NestedAggregation * max(len(nested), 1))(*nested)
    nbufs = [np.zeros(nq * 2048, np.float64) for _ in nested]
    nres = (_native.NestedResult * max(len(nested), 1))(*[_native.NestedResult(b.ctypes.data, None, None, None, None) for b in nbufs])
    docs, scores, counts, total = np.zeros((nq, k), np.int32), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32), np.zeros(nq, np.int64)
    try:
        _native.check(lib.nrtgpu_searcher_search_bool_aggs_nested(searcher, carr, ncl, qarr, nq, k, 0, arr, len(aggs), res, narr,
                                                                  len(nested), nres, C.c_void_p(0), docs.ctypes.data,
                                                                  scores.ctypes.data, counts.ctypes.data, total.ctypes.data))
    finally:
        raw.last = (docs, counts, total, bufs, nbufs)


def test_refusals(shard):
    sh, whole, _, searcher, _ = shard
    one = GpuIndexSearcher(whole)
    qs = QUERIES[:3]
    A, Nst = _native.Aggregation, _native.NestedAggregation

    def same_refusal(exc, status, msg, queries, adds, k=K):
        """the searcher refuses as the single image does"""
        for s in (searcher, one):
            with pytest.raises(exc) as e:
                s.search_with_collectors(queries, RelevanceCollector(k), adds)
            assert e.value.status == status and msg in e.value.message, e.value.message

    def refused(exc, status, msg, handle, queries, aggs, nested):
        with pytest.raises(exc) as e:
            raw(handle, queries, aggs, nested)
        assert e.value.status == status and msg in e.value.message, e.value.message
        docs, counts, total, bufs, nbufs = raw.last
        assert not docs.any() and not counts.any() and not total.any()
        assert not any(b.any() for b in bufs) and not any(b.any() for b in nbufs), "a refused call wrote an output"

    tree = BooleanQuery().add(BooleanQuery().add(TermQuery(5), Occur.SHOULD).add(TermQuery(9), Occur.SHOULD), Occur.MUST)
    same_refusal(NrtGpuUnsupported, 3, "nested BooleanQuery is outside the GPU path", [tree], [terms(C_INT, 3)])
    five = ta.bq(*[(ta.T(t), ta.S) for t in (5, 9, 20, 33, 50)])
    same_refusal(NrtGpuUnsupported, 3, "more than 4 term clauses or top_k > 512", [five], [terms(C_INT, 3)])
    same_refusal(NrtGpuUnsupported, 3, "more than 4 term clauses or top_k > 512", qs, [terms(C_INT, 3)], k=513)
    same_refusal(NrtGpuUnsupported, 3, "aggregation on a multi-valued column", qs, [MinCollector(MV)])
    same_refusal(NrtGpuUnsupported, 3, "aggregation on a multi-valued column", qs, [terms(MV, 3)])
    terms7 = A(1, C_INT, 0, 7, 1, 0)
    refused(NrtGpuError, 1, "NULL searcher", None, qs, [terms7], [])
    refused(NrtGpuError, 1, "no aggregations", searcher.handle, qs, [], [])
    for parent in (-1, 1):
        refused(NrtGpuError, 1, "parent out of range", searcher.handle, qs, [terms7], [Nst(parent, 3, F64, 2, 0, 0, 0, 0)])
    refused(NrtGpuError, 1, "aggregation column out of range", searcher.handle, qs, [A(1, len(sh.columns), 0, 7, 1, 0)], [])
    # the reader-wide tables: U = N distinct values of UNIQ, while no leaf holds more than 449,962
    nq = 2**29 // N + 1
    assert nq * (CUTS[3] - CUTS[2]) * 4 <= 2**31 < nq * N * 4
    refused(NrtGpuUnsupported, 3, "exceeds the 2 GB count table", searcher.handle, [MatchAllDocsQuery()] * nq, [A(1, UNIQ, 0, 1, 1, 0)], [])
    nq = 2**28 // N + 1
    refused(NrtGpuUnsupported, 3, "exceeds the 2 GB table", searcher.handle, [MatchAllDocsQuery()] * nq, [A(1, UNIQ, 0, 1, 1, 0)],
            [Nst(0, 3, C_INT, 0, 0, 0, 0, 0)])
    # the searcher still answers
    _, outs = searcher.search_with_collectors(qs, RelevanceCollector(K), [ta.stat(MaxCollector, C_INT)])
    assert outs[0].tolist() == [29.0] * 3
