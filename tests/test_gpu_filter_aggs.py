"""Filter collectors (nrtgpu_search_bool_aggs_filtered, FilterCollector) against tests/filter_aggs_reference.py over the
oracle's match sets and scores.

The shard is the 1.1M-doc aggregation shard of tests/test_gpu_aggregations.py (three probe slices, split parts, every 11th
doc deleted), moved to doc_base 1000; the batch mixes pure disjunctions, conjunctions, dense-driver and empty queries. Filters
are flat queries (term, range and multi-valued range clauses, MUST_NOT) and value sets on int, long, float and double columns
and on the multi-valued column, nested in each other. docCount, terms buckets, MIN / MAX and top hits (docs and score bits)
are exact, SUM within n * 2^-53 * sum|v|. The request's hits, totalHits and sibling aggregations equal a run without the
filter collectors; a terms aggregation under a one-clause filter equals the unfiltered path's terms aggregation of the query
with that clause added as FILTER; three leaves of a GpuLeafSearcher give what one image of the whole shard gives."""
import ctypes as C
import math

import numpy as np
import pytest

import filter_aggs_reference as fr
import nested_aggs_reference as nr
import oracle
from nrtsearch_b200 import NrtGpuError, NrtGpuUnsupported
from nrtsearch_b200 import _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, FilterCollector, GpuIndex, GpuIndexSearcher, GpuLeafSearcher, MatchAllDocsQuery,
                                   MaxCollector, MinCollector, Occur, RangeQuery, RelevanceCollector, SumCollector, TermQuery,
                                   TermsCollector, TopHitsCollector, ValueSetFilter, _FilteredRecords, compile_queries)
from test_gpu_aggregations import (C_INT, D2047, F32, F64, FIELD_TYPE, I64, MV, N, QUERIES, SEL, SEL_NAN, VALUE_TYPE, VOCAB,
                                   make_columns)

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
K = 20
DOC_BASE = 1000
S, M_, F, NOT = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
KIND = {MinCollector: "min", MaxCollector: "max", SumCollector: "sum"}
# simple and generic disjunctions, a conjunction with a range, MUST_NOT, msm, match-all, dense-driver ranges, empty queries
BATCH = [QUERIES[i] for i in (0, 1, 4, 5, 7, 8, 9, 10, 12, 13, 15, 16, 17, 22)]


@pytest.fixture(scope="module")
def big(gpu_ctx):
    sh = ix.synth_text_shard(N, VOCAB, seed=0xA66, min_len=4, poisson_mean=10.0)
    sh.columns, sh.column_has, offs = make_columns(N, 0xA67)
    sh.column_offsets = [None] * MV + [offs]
    sh.live_docs = (np.arange(N) % 11 != 0).astype(np.uint8)
    sh.doc_base = DOC_BASE
    gix = GpuIndex(gpu_ctx, sh)
    yield sh, gix, oracle.OracleIndex(sh)
    gix.close()


class Ref:
    """match sets, oracle scores and filter masks of a batch on one shard, computed once"""

    def __init__(self, sh, oix, queries):
        self.sh, self.oix = sh, oix
        self.carr, _, self.qarr, nq = compile_queries(queries)
        self.match = [oracle.match_bitmap(oix, self.carr, self.qarr, q).astype(bool) for q in range(nq)]
        self._scores, self._masks = {}, {}

    def scores(self, q):
        if q not in self._scores:
            self._scores[q] = nr.query_scores(self.sh, self.oix, self.carr, self.qarr, q, self.match[q])
        return self._scores[q]

    def mask(self, f):
        key = repr(f)
        if key not in self._masks:
            if isinstance(f, ValueSetFilter):
                self._masks[key] = fr.value_set_mask(self.sh, f.column, f.sortable())
            else:
                carr, _, qarr, _ = compile_queries([f])
                self._masks[key] = fr.query_mask(self.oix, carr, qarr, 0)
        return self._masks[key]

    def spec(self, c):
        if isinstance(c, TermsCollector):
            return ("terms", c.column, c.size, c.order_desc, {n: self.spec(x) for n, x in c.nested}, c.order_by)
        if isinstance(c, FilterCollector):
            return ("filter", self.mask(c.filter), {n: self.spec(x) for n, x in c.nested})
        if isinstance(c, TopHitsCollector):
            return ("top_hits", c.top_hits, c.start_hit)
        return (KIND[type(c)], c.column, VALUE_TYPE[c.field_type])


def has_top_hits(c):
    return isinstance(c, TopHitsCollector) or any(has_top_hits(x) for _, x in getattr(c, "nested", ()))


def close_sum(g, v, bound):
    return v is None or (math.isnan(v) and math.isnan(g)) or g == v or abs(g - v) <= bound


def check_value(g, spec, v, bound, what):
    if spec[0] == "sum":
        assert close_sum(g, v, bound), f"{what}: {g!r} vs {v!r} +- {bound}"
    else:
        assert g == v or (math.isnan(g) and math.isnan(v)), f"{what}: {g!r} vs {v!r}"


def check_terms(o, w, spec, q, what):
    _, _, size, _, sub, _ = spec
    assert o["n"][q] == w["n"] and o["total_buckets"][q] == w["total_buckets"], what
    assert o["other_counts"][q] == w["other_counts"], what
    assert np.array_equal(o["keys"][q], w["keys"]) and np.array_equal(o["counts"][q], w["counts"]), what
    n = w["n"]
    for name, s in sub.items():
        got = o["nested"][name]
        if s[0] == "top_hits":
            for b, (docs, scores, total) in enumerate(w["nested"][name]):
                m = len(docs)
                assert got["counts"][q, b] == m and got["total_hits"][q, b] == total, f"{what} {name} slot {b}"
                assert got["docs"][q, b, :m].tolist() == docs.tolist(), f"{what} {name} slot {b}: docs"
                assert np.array_equal(got["scores"][q, b, :m].view(np.uint32), scores.view(np.uint32)), f"{what} {name} slot {b}"
            assert not got["counts"][q, n:].any()
        else:
            for b, (v, bound) in enumerate(w["nested"][name]):
                check_value(float(got[q, b]), s, v, bound, f"{what} {name} slot {b}")
            assert not got[q, n:].any()


def check_filter(o, w, spec, q, what):
    assert o["doc_count"][q] == w["doc_count"], f"{what}: docCount {o['doc_count'][q]} vs {w['doc_count']}"
    for name, s in spec[2].items():
        got, want, at = o[name], w[name], f"{what} / {name}"
        if s[0] == "terms":
            check_terms(got, want, s, q, at)
        elif s[0] == "filter":
            check_filter(got, want, s, q, at)
        elif s[0] == "top_hits":
            docs, scores, total = want
            m = len(docs)
            assert got["counts"][q] == m and got["total_hits"][q] == total, at
            assert got["docs"][q, :m].tolist() == docs.tolist(), f"{at}: docs"
            assert np.array_equal(got["scores"][q, :m].view(np.uint32), scores.view(np.uint32)), f"{at}: scores"
            assert not got["docs"][q, m:].any()
        else:
            check_value(float(got[q]), s, want[0], want[1], at)


def check_all(ref, adds, outs, rows=None):
    for a, o in zip(adds, outs):
        if not isinstance(a, FilterCollector):
            continue
        spec = ref.spec(a)
        scores = has_top_hits(a)
        for q in (range(len(ref.match)) if rows is None else rows):
            sel = ref.match[q] & spec[1]
            w = fr.filter_result(ref.sh, sel, spec[2], ref.scores(q) if scores else None)
            check_filter(o, w, spec, q, f"query {q}")


def T(t):
    return TermQuery(t)


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(c, o)
    return q


def terms(c, size, desc=True, nested=(), order_by=None):
    return TermsCollector(c, size, desc, FIELD_TYPE[c], tuple(nested), order_by)


def stat(cls, c):
    return cls(c, FIELD_TYPE[c])


# a query filter of term, range and multi-valued range clauses; a value set on the multi-valued column under it
QFILTER = bq((T(1), S), (RangeQuery(I64, 0, 2**62), S), (RangeQuery(MV, 10, 30), S), (T(3), NOT))
MAIN = [
    terms(C_INT, 12),                                                   # a sibling without a filter
    FilterCollector(QFILTER, nested=(
        ("by_int", terms(C_INT, 10, nested=(("mx", stat(MaxCollector, F64)), ("th", TopHitsCollector(5))))),
        ("min_f32", stat(MinCollector, F32)),
        ("sum_int", stat(SumCollector, C_INT)),
        ("hits", TopHitsCollector(7, 2)),
        ("mv", FilterCollector(ValueSetFilter(MV, (7, 14, 21, 56, 10**6)), nested=(
            ("by_2047", terms(D2047, 6, False, nested=(("mn", stat(MinCollector, F32)),), order_by="mn")),
            ("max_i64", stat(MaxCollector, I64)),
            ("top", TopHitsCollector(3)))),
         ),
    )),
    stat(SumCollector, F64),
]


def search(gix, queries, adds, k=K):
    return GpuIndexSearcher(gix).search_with_collectors(queries, RelevanceCollector(k, INT_MAX), adds)


def same_hits(a, b):
    assert np.array_equal(a.docs, b.docs) and np.array_equal(a.counts, b.counts)
    assert np.array_equal(a.scores.view(np.uint32), b.scores.view(np.uint32))
    assert np.array_equal(a.total_hits, b.total_hits)


@pytest.fixture(scope="module")
def ref(big):
    sh, _, oix = big
    return Ref(sh, oix, BATCH)


def test_filters_against_the_reference(big, ref):
    _, gix, _ = big
    res, outs = search(gix, BATCH, MAIN)
    check_all(ref, MAIN, outs)
    # the hits, totalHits and the sibling collectors are those of the same call without the filter collector
    plain, plain_outs = search(gix, BATCH, [MAIN[0], MAIN[2]])
    same_hits(res, plain)
    assert all(np.array_equal(outs[0][x], plain_outs[0][x]) for x in plain_outs[0])
    assert np.array_equal(outs[2].view(np.uint64), plain_outs[1].view(np.uint64))
    # a repeated call is identical
    again, again_outs = search(gix, BATCH, MAIN)
    same_hits(res, again)
    assert repr(again_outs) == repr(outs)


def test_value_sets_of_every_column_type(big, ref):
    _, gix, _ = big
    nested = (("s", stat(MaxCollector, C_INT)),)
    f32 = [float(np.float32(x)) for x in (-0.0, math.nan, 1e-45)]
    adds = [FilterCollector(ValueSetFilter(C_INT, (-30, 0, 29, 29, 5, 1000), "int"), nested),
            FilterCollector(ValueSetFilter(I64, (-2**63, 2**63 - 1, 0, -1, 2**62), "long"), nested),
            FilterCollector(ValueSetFilter(F32, tuple(f32), "float"), nested),
            FilterCollector(ValueSetFilter(F64, (0.0, math.nan, -math.inf, 5e-324), "double"), nested),
            FilterCollector(ValueSetFilter(MV, (8, 15, 64, 57), "long"), nested),
            FilterCollector(ValueSetFilter(SEL, (), "int"), nested),         # the empty set passes nothing
            FilterCollector(ValueSetFilter(F64, (-0.0,), "double"), nested)]
    _, outs = search(gix, BATCH, adds)
    check_all(ref, adds, outs)
    assert not outs[5]["doc_count"].any()
    assert outs[3]["doc_count"][BATCH.index(QUERIES[17])] > 0   # the NaN docs of "only NaN" pass a set holding NaN
    assert (ref.sh.columns[SEL] == SEL_NAN).any()


def with_filter(q, clause):
    """q AND clause, as a flat BooleanQuery matching exactly what q matches and clause matches"""
    if not isinstance(q, BooleanQuery):
        return bq((q, M_), (clause, F))
    if not q.clauses:
        return q
    required = any(c.occur in (Occur.MUST, Occur.FILTER) for c in q.clauses)
    msm = q.minimum_number_should_match if required else max(q.minimum_number_should_match, 1)
    return bq(*[(c.query, c.occur) for c in q.clauses], (clause, F), msm=msm)


@pytest.mark.parametrize("clause", [RangeQuery(C_INT, -10, 10), RangeQuery(MV, 0, 20), RangeQuery(I64, -2**61, 2**62)])
def test_terms_under_one_clause_filter_equals_the_filtered_query(big, clause):
    _, gix, _ = big
    t = terms(D2047, 8, nested=(("mx", stat(MaxCollector, C_INT)),))
    _, outs = search(gix, BATCH, [FilterCollector(clause, (("t", t),))])
    _, want = search(gix, [with_filter(q, clause) for q in BATCH], [t])
    got = outs[0]["t"]
    for x in ("keys", "counts", "n", "total_buckets", "other_counts"):
        assert np.array_equal(got[x], want[0][x]), x
    assert np.array_equal(got["nested"]["mx"].view(np.uint64), want[0]["nested"]["mx"].view(np.uint64))


def test_three_leaves_equal_one_image(gpu_ctx, big, ref):
    sh, gix, _ = big
    cuts = [0, 300_001, 300_038, N]   # a leaf of 37 docs, a cut inside a probe slice
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(lo, hi, doc_base=DOC_BASE + lo)) for lo, hi in zip(cuts, cuts[1:])]
    s = GpuLeafSearcher(gpu_ctx, leaves)
    try:
        res, outs = s.search_with_collectors(BATCH, RelevanceCollector(K, INT_MAX), MAIN)
        one, one_outs = search(gix, BATCH, MAIN)
        same_hits(res, one)
        check_all(ref, MAIN, outs)

        def exact(a, b):   # everything but the sums, whose order differs between the leaves and the image
            if isinstance(a, dict):
                for x in a:
                    if x not in ("sum_int",):
                        exact(a[x], b[x])
            else:
                assert np.array_equal(a, b)
        exact(outs[1], one_outs[1])
    finally:
        s.close()
        for g in leaves:
            g.close()


def raw_call(gix, queries, adds, fill):
    """the single-image entry point with pre-filled outputs: (status, every output array)"""
    carr, ncl, qarr, nq = compile_queries(queries)
    rec = _FilteredRecords(nq, adds)
    hits = [np.full((nq, K), fill, np.int32), np.full((nq, K), fill, np.float32), np.full(nq, fill, np.int32),
            np.full(nq, fill, np.int64)]
    arrays = list(hits)

    def collect(o):
        if isinstance(o, dict):
            for v in o.values():
                collect(v)
        else:
            o[...] = fill
            arrays.append(o)
    for o in rec.outs:
        collect(o)
    rc = _native.gpu_lib().nrtgpu_search_bool_aggs_filtered(gix.handle, carr, ncl, qarr, nq, K, 0, *rec.args, None,
                                                            *[h.ctypes.data for h in hits])
    return rc, arrays


def test_refused_calls_write_nothing(big):
    sh, gix, _ = big
    wide = BooleanQuery()
    for i in range(17):
        wide.add(RangeQuery(C_INT, i, i), Occur.SHOULD)
    cases = [([FilterCollector(T(5), ())], 1, 'Filter collector "aggs[0]" must have nested collectors'),
             ([FilterCollector(wide, (("m", stat(MinCollector, C_INT)),))], 3, "more than 16 clauses"),
             ([FilterCollector(T(5), (("t", TermsCollector(MV, 4)),))], 3, "aggregation on a multi-valued column"),
             ([FilterCollector(ValueSetFilter(40, (1,)), (("m", stat(MinCollector, C_INT)),))], 1, "column out of range")]
    for adds, code, msg in cases:
        rc, arrays = raw_call(gix, BATCH, adds, 7)
        assert rc == code, msg
        assert msg in _native.gpu_lib().nrtgpu_last_error().decode()
        assert all((a == 7).all() for a in arrays), msg
    with pytest.raises(NrtGpuError):
        search(gix, BATCH, [FilterCollector(T(5), ())])
    with pytest.raises(NrtGpuUnsupported):
        search(gix, BATCH, [FilterCollector(wide, (("m", stat(MinCollector, C_INT)),))])
    with pytest.raises(ValueError):   # a filter collector under a terms collector stays refused
        search(gix, BATCH, [terms(C_INT, 3, nested=(("f", FilterCollector(T(5), (("m", stat(MinCollector, C_INT)),))),))])
    res, outs = search(gix, BATCH[:3], [FilterCollector(T(5), (("m", stat(MinCollector, C_INT)),))])   # the index answers
    assert res.counts.any() and outs[0]["doc_count"].any()


def test_live_docs_updates_are_followed(gpu_ctx):
    n = 300_000
    sh = ix.synth_text_shard(n, 3000, seed=5)
    rng = np.random.default_rng(6)
    sh.columns = [rng.integers(0, 50, n).astype(np.int64), rng.integers(0, 7, n).astype(np.int64)]
    sh.column_has = [None, None]
    queries = [MatchAllDocsQuery(), bq((T(0), S), (T(1), S)), RangeQuery(0, 10, 40)]
    adds = [FilterCollector(ValueSetFilter(1, (2, 3)), (("t", terms(0, 5)), ("h", TopHitsCollector(4)))),
            FilterCollector(bq((T(2), S), (RangeQuery(0, 0, 9), S)), (("s", SumCollector(1)),))]
    gix = GpuIndex(gpu_ctx, sh)
    try:
        for live in (None, (np.arange(n) % 3 != 0).astype(np.uint8), (rng.random(n) < 0.5).astype(np.uint8)):
            sh.live_docs = live
            gix.set_live_docs(live)
            ref = Ref(sh, oracle.OracleIndex(sh), queries)
            _, outs = search(gix, queries, adds)
            check_all(ref, adds, outs)
    finally:
        gix.close()


def test_knn_filter_stats_survive_an_aggregation_call(gpu_ctx):
    from test_gpu_knn_filter import filter_shard
    sh = filter_shard(20_000, 32, ix.SIM_COSINE, seed=3)
    queries = ix.synth_vectors(8, 32, seed=9)
    flt = [TermQuery(0), RangeQuery(0, 0, 3), None, RangeQuery(1, 5, 6), TermQuery(1), None, MatchAllDocsQuery(), TermQuery(0)]
    gix = GpuIndex(gpu_ctx, sh)
    lib = _native.gpu_lib()

    def stats():
        g, ms = C.c_int32(), C.c_float()
        assert lib.nrtgpu_knn_filter_stats(gix.handle, C.byref(g), C.byref(ms)) == 0
        return g.value, ms.value
    try:
        s = GpuIndexSearcher(gix)
        first = s.knn(queries, 10, filter_queries=flt)
        before = stats()
        _, outs = s.search_with_collectors([MatchAllDocsQuery()], RelevanceCollector(5, INT_MAX),
                                           [FilterCollector(bq((T(0), S), (RangeQuery(1, 0, 9), S)), (("m", MaxCollector(2)),))])
        assert outs[0]["doc_count"][0] > 0
        assert stats() == before
        second = s.knn(queries, 10, filter_queries=flt)
        for a, b in zip(first, second):
            assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))
        assert stats()[0] == before[0]
    finally:
        gix.close()
