"""Nested collectors of terms aggregations (nrtgpu_search_bool_aggs_nested: per-bucket min / max / sum and top hits, buckets
ordered by a nested value) against tests/nested_aggs_reference.py over the oracle's match sets and scores.

Two shards: the 100-doc known-answer shard of NestedCollectorOrderTest / NestedCollectionTest, and the 1.1M-doc shard of
tests/test_gpu_aggregations.py (three probe slices, split parts, dense-driver queries, every 11th doc deleted) moved to
doc_base 1000, with its count ties, 2047 / 2048 / 2049 distinct values around the 2048-bucket chunk, missing values, NaN,
+-inf and +-0. Keys, counts, MIN / MAX and top hits (docs and score bits) are exact, SUM within n * 2^-53 * sum|v|; the
request's hits, totalHits and sibling aggregations equal a run without the nested collectors."""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest

import nested_aggs_reference as nr
import oracle
from helpers import shard_from_token_docs
from nrtsearch_b200 import NrtGpuError, NrtGpuUnsupported
from nrtsearch_b200 import _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (GpuIndex, GpuIndexSearcher, MatchAllDocsQuery, MaxCollector, MinCollector, RangeQuery,
                                   RelevanceCollector, SumCollector, TermQuery, TermsCollector, TopHitsCollector,
                                   compile_queries)
from test_gpu_aggregations import (C_INT, D2047, D2048, D2049, F32, F64, FIELD_TYPE, I64, MV, N, NONE, QUERIES, SEL, UNIQ,
                                   VALUE_TYPE, VOCAB, make_columns)

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
K = 50
DOC_BASE = 1000
KIND = {MinCollector: "min", MaxCollector: "max", SumCollector: "sum"}


@pytest.fixture(scope="module")
def big(gpu_ctx):
    sh = ix.synth_text_shard(N, VOCAB, seed=0xA66, min_len=4, poisson_mean=10.0)
    sh.columns, sh.column_has, offs = make_columns(N, 0xA67)
    sh.column_offsets = [None] * MV + [offs]
    sh.live_docs = (np.arange(N) % 11 != 0).astype(np.uint8)
    sh.doc_base = DOC_BASE
    gix = GpuIndex(gpu_ctx, sh)
    oix = oracle.OracleIndex(sh)
    yield sh, gix, oix
    gix.close()


class Ref:
    """match sets and oracle scores of a batch on one shard, computed once"""

    def __init__(self, sh, oix, queries):
        self.sh = sh
        self.carr, _, self.qarr, nq = compile_queries(queries)
        self.match = [oracle.match_bitmap(oix, self.carr, self.qarr, q).astype(bool) for q in range(nq)]
        self.oix = oix
        self._scores = {}

    def scores(self, q):
        if q not in self._scores:
            self._scores[q] = nr.query_scores(self.sh, self.oix, self.carr, self.qarr, q, self.match[q])
        return self._scores[q]


def spec(c):
    if isinstance(c, TopHitsCollector):
        return ("top_hits", c.top_hits, c.start_hit)
    return (KIND[type(c)], c.column, VALUE_TYPE[c.field_type])


def check_terms(ref, a, o, rows=None):
    """one terms collector's result (with its nested results) against the reference, query by query"""
    nested = {name: spec(c) for name, c in a.nested}
    need_scores = any(s[0] == "top_hits" for s in nested.values())
    for q in (range(len(ref.match)) if rows is None else rows):
        w = nr.terms_nested(ref.sh, ref.match[q], a.column, a.size, a.order_desc, nested, a.order_by,
                            ref.scores(q) if need_scores else None)
        what = f"query {q}, terms column {a.column} size {a.size}"
        assert o["n"][q] == w["n"] and o["total_buckets"][q] == w["total_buckets"], what
        assert o["other_counts"][q] == w["other_counts"], what
        assert np.array_equal(o["keys"][q], w["keys"]) and np.array_equal(o["counts"][q], w["counts"]), what
        n = w["n"]
        for name, s in nested.items():
            got = o["nested"][name]
            if s[0] == "top_hits":
                top, start = s[1], s[2]
                for b, (docs, scores, total) in enumerate(w["nested"][name]):
                    m = len(docs)
                    assert got["counts"][q, b] == m and got["total_hits"][q, b] == total, f"{what} {name} slot {b}"
                    assert got["docs"][q, b, :m].tolist() == docs.tolist(), f"{what} {name} slot {b}: docs"
                    assert np.array_equal(got["scores"][q, b, :m].view(np.uint32), scores.view(np.uint32)), f"{what} {name} slot {b}: scores"
                    assert not got["docs"][q, b, m:].any()
                assert not got["counts"][q, n:].any() and not got["total_hits"][q, n:].any()
                assert got["docs"].shape[2] == top - start
                continue
            for b, (v, bound) in enumerate(w["nested"][name]):
                g = float(got[q, b])
                if s[0] == "sum":
                    if v is None:   # some summation order overflows: any result is one of them
                        continue
                    ok = (math.isnan(v) and math.isnan(g)) or g == v or abs(g - v) <= bound
                    assert ok, f"{what} {name} slot {b}: {g!r} vs {v!r} +- {bound}"
                else:
                    assert g == v, f"{what} {name} slot {b}: {g!r} vs {v!r}"
            assert not got[q, n:].any()


def strip(adds):
    return [dataclasses.replace(a, nested=(), order_by=None) if isinstance(a, TermsCollector) else a for a in adds]


def search_and_check(gix, ref, queries, adds, k=K):
    s = GpuIndexSearcher(gix)
    res, outs = s.search_with_collectors(queries, RelevanceCollector(k, INT_MAX), adds)
    plain, plain_outs = s.search_with_collectors(queries, RelevanceCollector(k, INT_MAX), strip(adds))
    assert np.array_equal(res.docs, plain.docs) and np.array_equal(res.counts, plain.counts)
    assert np.array_equal(res.scores.view(np.uint32), plain.scores.view(np.uint32))
    assert np.array_equal(res.total_hits, plain.total_hits)
    for a, o, p in zip(adds, outs, plain_outs):
        if isinstance(a, TermsCollector):
            if a.order_by is None:   # ordered by count: the same buckets as without the nested collectors
                assert all(np.array_equal(o[x], p[x]) for x in p)
            check_terms(ref, a, o)
        else:
            assert np.array_equal(o.view(np.uint64), p.view(np.uint64))
    return res, outs


def terms(c, size, desc=True, nested=(), order_by=None):
    return TermsCollector(c, size, desc, FIELD_TYPE[c], tuple(nested), order_by)


def stat(cls, c):
    return cls(c, FIELD_TYPE[c])


# ---------------------------------------------------------------- the known-answer shard (NestedCollectorOrderTest)
def test_known_answers(gpu_ctx):
    i, j = np.repeat(np.arange(1, 6), 20), np.tile(np.arange(1, 21), 5)
    docs = [["a"] * (1 + d // 10) + ["b"] * (9 - d // 10) for d in range(100)]
    ids = np.arange(100, dtype=np.int64)
    sh, vocab = shard_from_token_docs([docs], columns=[i.astype(np.int64), (i * j).astype(np.int64), (-i * j).astype(np.int64),
                                                       ids % 2])
    gix = GpuIndex(gpu_ctx, sh)
    try:
        s = GpuIndexSearcher(gix)
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
        # NestedCollectionTest: two buckets of 50, top 5 hits each, totalHits 50
        a = TermsCollector(3, 2, True, "int", (("nested", TopHitsCollector(5)),))
        res, outs = s.search_with_collectors([TermQuery(vocab[(0, "a")])], RelevanceCollector(10), [a])
        o = outs[0]
        assert sorted(o["keys"][0].tolist()) == [0, 1] and o["counts"][0].tolist() == [50, 50]
        h = o["nested"]["nested"]
        for b, key in enumerate(o["keys"][0].tolist()):
            assert h["total_hits"][0, b] == 50 and h["counts"][0, b] == 5
            assert h["docs"][0, b].tolist() == [90 + key, 92 + key, 94 + key, 96 + key, 98 + key]
            assert h["scores"][0, b].view(np.uint32).tolist() == [res.scores[0, 0].view(np.uint32)] * 5
        check_terms(Ref(sh, oracle.OracleIndex(sh), [TermQuery(vocab[(0, "a")])]), a, o)
    finally:
        gix.close()


# ---------------------------------------------------------------- the 1.1M-doc shard
@pytest.fixture(scope="module")
def ref(big):
    sh, _, oix = big
    return Ref(sh, oix, QUERIES)


GROUPS = [
    # count ties (60 equal shares), every metric kind on float / double / int64 columns with NaN, +-inf, +-0, missing values
    [terms(C_INT, 7, nested=[("max", stat(MaxCollector, F64)), ("min", stat(MinCollector, F32)), ("sum", stat(SumCollector, I64)),
                             ("hits", TopHitsCollector(10))]),
     terms(C_INT, 7, False, nested=[("sum", stat(SumCollector, SEL)), ("hits", TopHitsCollector(4, 3))]),
     stat(MaxCollector, F64), terms(SEL, 6), stat(SumCollector, C_INT)],
    # ordered by a nested value around the 2048-bucket chunk, both directions; top hits larger than small buckets
    [terms(D2049, 2048, nested=[("max", stat(MaxCollector, F64)), ("hits", TopHitsCollector(3, 1))], order_by="max"),
     terms(D2047, 2047, False, nested=[("min", stat(MinCollector, F32))], order_by="min"),
     terms(D2048, 5, nested=[("sum", stat(SumCollector, C_INT)), ("max", stat(MaxCollector, I64))], order_by="sum"),
     terms(D2048, 7, False, nested=[("sum", stat(SumCollector, C_INT))], order_by="sum")],
    # ties of the order value (SEL buckets share +-inf / MAX maxima, NONE has no values at all) and large top hits
    [terms(SEL, 6, nested=[("max", stat(MaxCollector, F32)), ("hits", TopHitsCollector(1024, 2))], order_by="max"),
     terms(SEL, 4, False, nested=[("max", stat(MaxCollector, F32))], order_by="max"),
     terms(C_INT, 60, nested=[("none", stat(MaxCollector, NONE))], order_by="none"),
     terms(C_INT, 3, False, nested=[("none", stat(MinCollector, NONE))], order_by="none")],
]


@pytest.mark.parametrize("group", range(len(GROUPS)))
def test_nested_match_reference(big, ref, group):
    _, gix, _ = big
    search_and_check(gix, ref, QUERIES, GROUPS[group])


def test_top_hits_in_query_groups(big):
    """80 queries whose returned buckets hold every live doc: 80M keys, more than one pass-2 group of 2^26"""
    sh, gix, oix = big
    qs = [RangeQuery(C_INT, -30, 30)] * 80
    a = terms(C_INT, 60, nested=[("hits", TopHitsCollector(5)), ("max", stat(MaxCollector, F64))])
    r = Ref(sh, oix, qs[:1])
    s = GpuIndexSearcher(gix)
    res, outs = s.search_with_collectors(qs, RelevanceCollector(10, INT_MAX), [a])
    assert res.total_hits[0] * 80 > 2**26
    check_terms(r, a, outs[0], rows=[0])
    o = outs[0]
    for q in range(1, 80):
        assert np.array_equal(o["keys"][q], o["keys"][0])
        for x in ("docs", "counts", "total_hits"):
            assert np.array_equal(o["nested"]["hits"][x][q], o["nested"]["hits"][x][0]), (q, x)
        assert np.array_equal(o["nested"]["hits"]["scores"][q].view(np.uint32), o["nested"]["hits"]["scores"][0].view(np.uint32))


def test_repeated_call_is_identical(big):
    """everything but the sums, whose atomics add in an order that may differ from call to call"""
    _, gix, _ = big
    s = GpuIndexSearcher(gix)
    adds = GROUPS[0]
    _, o1 = s.search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX), adds)
    _, o2 = s.search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX), adds)
    for a, x, y in zip(adds, o1, o2):
        if isinstance(a, TermsCollector):
            assert all(np.array_equal(x[f], y[f]) for f in ("keys", "counts", "n", "total_buckets", "other_counts"))
            for name, c in a.nested:
                gx, gy = x["nested"][name], y["nested"][name]
                if isinstance(c, TopHitsCollector):
                    assert all(np.array_equal(gx[f], gy[f]) for f in ("docs", "counts", "total_hits"))
                    assert np.array_equal(gx["scores"].view(np.uint32), gy["scores"].view(np.uint32))
                elif not isinstance(c, SumCollector):
                    assert np.array_equal(gx.view(np.uint64), gy.view(np.uint64))


def raw_nested(gix, queries, aggs, nested, k=K):
    """nrtgpu_search_bool_aggs_nested with hand-made records"""
    lib = _native.gpu_lib()
    carr, ncl, qarr, nq = compile_queries(queries)
    arr = (_native.Aggregation * len(aggs))(*aggs)
    bufs = [(np.zeros(nq * a.size, np.int64), np.zeros(nq * a.size, np.int32), np.zeros(nq, np.int32), np.zeros(nq, np.int32),
             np.zeros(nq, np.int64)) for a in aggs]
    res = (_native.AggregationResult * len(aggs))(*[_native.AggregationResult(None, *[b.ctypes.data for b in bb]) for bb in bufs])
    narr = (_native.NestedAggregation * max(len(nested), 1))(*nested)
    nbufs = [np.zeros(nq * 2048 * 8, np.float64) for _ in nested]
    nres = (_native.NestedResult * max(len(nested), 1))(*[_native.NestedResult(b.ctypes.data, None, None, None, None) for b in nbufs])
    docs, scores, counts, total = np.zeros((nq, k), np.int32), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32), np.zeros(nq, np.int64)
    _native.check(lib.nrtgpu_search_bool_aggs_nested(gix.handle, carr, ncl, qarr, nq, k, 0, arr, len(aggs), res, narr, len(nested),
                                                     nres, C.c_void_p(0), docs.ctypes.data, scores.ctypes.data, counts.ctypes.data,
                                                     total.ctypes.data))
    return docs, scores, counts, total, bufs


def test_no_nested_is_the_aggregation_entry(big):
    _, gix, _ = big
    A = _native.Aggregation
    aggs = [A(1, C_INT, 0, 7, 1, 0), A(3, F64, 2, 0, 0, 0)]
    got = raw_nested(gix, QUERIES, aggs, [])
    res, outs = GpuIndexSearcher(gix).search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX),
                                                             [terms(C_INT, 7), stat(MaxCollector, F64)])
    assert np.array_equal(got[0], res.docs) and np.array_equal(got[1].view(np.uint32), res.scores.view(np.uint32))
    assert np.array_equal(got[2], res.counts) and np.array_equal(got[3], res.total_hits)
    assert np.array_equal(got[4][0][0].reshape(-1, 7), outs[0]["keys"]) and np.array_equal(got[4][0][1].reshape(-1, 7), outs[0]["counts"])


def test_refusals(big):
    sh, gix, _ = big
    qs = QUERIES[:3]
    A, Nst = _native.Aggregation, _native.NestedAggregation
    terms7 = A(1, C_INT, 0, 7, 1, 0)

    def refused(exc, status, msg, aggs, nested, queries=qs):
        with pytest.raises(exc) as e:
            raw_nested(gix, queries, aggs, nested)
        assert e.value.status == status and msg in e.value.message, e.value.message

    for parent in (-1, 2):
        refused(NrtGpuError, 1, "parent out of range", [terms7, A(2, C_INT, 0, 0, 0, 0)], [Nst(parent, 2, F64, 2, 0, 0, 0, 0)])
    refused(NrtGpuError, 1, "the parent is not a terms aggregation", [terms7, A(2, C_INT, 0, 0, 0, 0)], [Nst(1, 2, F64, 2, 0, 0, 0, 0)])
    for kind in (0, 1, 6):
        refused(NrtGpuError, 1, "bad nested aggregation kind", [terms7], [Nst(0, kind, F64, 2, 0, 0, 0, 0)])
    for col in (-1, len(sh.columns)):
        refused(NrtGpuError, 1, "nested aggregation column out of range", [terms7], [Nst(0, 3, col, 0, 0, 0, 0, 0)])
    for vt in (-1, 3):
        refused(NrtGpuError, 1, "bad nested aggregation value_type", [terms7], [Nst(0, 3, F64, vt, 0, 0, 0, 0)])
    for top, start in ((5, -1), (5, 5), (0, 0)):
        refused(NrtGpuError, 1, "start_hit must be in [0, top_hits)", [terms7], [Nst(0, 5, 0, 0, top, start, 0, 0)])
    refused(NrtGpuError, 1, "two collectors order one terms aggregation", [terms7],
            [Nst(0, 3, F64, 2, 0, 0, 1, 0), Nst(0, 2, F32, 1, 0, 0, 1, 0)])
    refused(NrtGpuError, 1, "top hits cannot order the buckets", [terms7], [Nst(0, 5, 0, 0, 5, 0, 1, 0)])
    refused(NrtGpuUnsupported, 3, "more than 4 nested aggregations", [terms7], [Nst(0, 3, F64, 2, 0, 0, 0, 0)] * 5)
    refused(NrtGpuUnsupported, 3, "nested aggregation on a multi-valued column", [terms7], [Nst(0, 3, MV, 0, 0, 0, 0, 0)])
    refused(NrtGpuUnsupported, 3, "top_hits > 1024", [terms7], [Nst(0, 5, 0, 0, 1025, 0, 0, 0)])
    # 9 x 2048 x 1024 outputs of one collector: over 2^24 (8 queries would be exactly 2^24)
    refused(NrtGpuUnsupported, 3, "exceeds 2^24 hits", [A(1, C_INT, 0, 2048, 1, 0)], [Nst(0, 5, 0, 0, 1024, 0, 0, 0)], QUERIES[:9])
    raw_nested(gix, QUERIES[:8], [A(1, C_INT, 0, 2048, 1, 0)], [Nst(0, 5, 0, 0, 1024, 1023, 0, 0)])
    # a nested metric's table: nq x distinct values x 8 bytes over 2 GB, while the count table stays under its 2 GB
    nq = (2**28) // (N - N // 11) + 1
    with pytest.raises(NrtGpuUnsupported) as e:
        raw_nested(gix, [MatchAllDocsQuery()] * nq, [A(1, UNIQ, 0, 1, 1, 0)], [Nst(0, 3, C_INT, 0, 0, 0, 0, 0)], k=1)
    assert e.value.status == 3 and "exceeds the 2 GB table" in e.value.message, e.value.message
    # the index still answers afterwards
    _, outs = GpuIndexSearcher(gix).search_with_collectors(qs, RelevanceCollector(K), [terms(C_INT, 2, nested=[("m", stat(MaxCollector, C_INT))])])
    assert outs[0]["n"].tolist() == [2] * 3
    assert np.array_equal(outs[0]["nested"]["m"], outs[0]["keys"].astype(np.float64))   # a bucket's max of its own key


def test_python_refusals(big):
    _, gix, _ = big
    s = GpuIndexSearcher(gix)
    with pytest.raises(ValueError):
        s.search_with_collectors(QUERIES[:2], RelevanceCollector(K), [terms(C_INT, 3, nested=[("a", stat(MaxCollector, F64))], order_by="b")])
    with pytest.raises(ValueError):
        s.search_with_collectors(QUERIES[:2], RelevanceCollector(K), [terms(C_INT, 3, nested=[("a", terms(SEL, 2))])])
    with pytest.raises(NrtGpuError):
        s.search_with_collectors(QUERIES[:2], RelevanceCollector(K), [terms(C_INT, 3, nested=[("h", TopHitsCollector(3))], order_by="h")])
