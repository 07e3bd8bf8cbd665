"""Collectors on the window engine (nrtgpu_search_tree_aggs / nrtgpu_searcher_search_tree_aggs, the kAggs instantiations of
bool_window_kernel) against the existing references, fed with rescore_tree_reference.evaluate_all: the match set and float32
score of every query over every doc, deletes applied.

The shard is tests/test_gpu_phrase.py's: 1.25M docs (two window-engine slices) with term positions, 5 % deletes and
postings planted on both sides of window and slice edges, plus a 40-value int column with missing values, a double column
with NaN, +-inf, -0.0 and 0.0, and a multi-valued column. Batches hold nested bools with MUST_NOT and msm, multi_match
dismax at tie 0 and 0.3, exact and sloppy phrases, range and match-all leaves and a query that matches nothing, plus a
flat 6-term batch and a top_k 1024 batch. Bucket keys and counts, min / max, top-hit docs, score bits and sort values are
exact, sums within aggs_reference's bound; every page equals search_tree's bit for bit. Three leaves with a doc_base, cut
inside a window, equal the whole image; refused calls write nothing; no collector state leaks between calls."""
import ctypes as C
import math

import numpy as np
import pytest

import aggs_reference as ar
import filter_aggs_reference as far
import nested_aggs_reference as nr
import oracle
import rescore_tree_reference as rtr
import searcher_leaves as sl
import sorted_hits_reference as shr
from nrtsearch_b200 import NrtGpuError, NrtGpuUnsupported
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, FilterCollector, GpuIndex, GpuIndexSearcher,
                                   GpuLeafSearcher, MatchAllDocsQuery, MaxCollector, MinCollector, Occur, RangeQuery,
                                   RelevanceCollector, SortType, SumCollector, TermQuery, TermsCollector, TopHitsCollector,
                                   ValueSetFilter, _FilteredRecords, compile_tree)
from test_gpu_phrase import A, B, C8, N_DOCS, PRICE, V0, WIDE_SLICE, P, bq, match, token_shard

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
CAT, DBL, MV = 1, 2, 3           # the added columns (0 is the price column)
VT = {"long": ar.INT, "int": ar.INT, "double": ar.DOUBLE}


def add_columns(sh):
    rng = np.random.default_rng(0x7A6)
    n = sh.n_docs
    cat = rng.integers(-5, 35, n).astype(np.int64)
    has_cat = (rng.random(n) >= 0.1).astype(np.uint8)
    pool = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, 1.5, -2.25, 1e300], np.float64)
    dv = np.where(rng.random(n) < 0.2, pool[rng.integers(0, len(pool), n)], np.round(rng.normal(0, 1e3, n), 2))
    b = dv.view(np.int64)
    dbl = b ^ ((b >> 63) & np.int64(0x7fffffffffffffff))   # NumericUtils.doubleToSortableLong
    per = rng.integers(0, 3, n)
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(per, out=offs[1:])
    owner = np.repeat(np.arange(n), per)
    vals = rng.integers(0, 50, int(offs[-1])).astype(np.int64)
    mv = vals[np.lexsort((vals, owner))]                    # ascending inside each doc (SORTED_NUMERIC)
    sh.columns = [sh.columns[0], cat, dbl, mv]
    sh.column_has = [None, has_cat, None, None]
    sh.column_offsets = [None, None, None, offs]
    return sh


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    sh = add_columns(token_shard())
    g = GpuIndex(gpu_ctx, sh)
    yield sh, oracle.OracleIndex(sh), g
    g.close()


@pytest.fixture(scope="module")
def leaves(gpu_ctx, corpus):
    sh = corpus[0]
    cuts = [0, 400_000 + 5_000, WIDE_SLICE + 3, N_DOCS]   # 405,000 is inside a 16,384-doc window
    ls = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    s = GpuLeafSearcher(gpu_ctx, ls)
    yield ls, s
    s.close()
    for g in ls:
        g.close()


def T(t):
    return TermQuery(int(t))


C1 = [V0 + 3, V0 + 5]   # a common field-1 bigram
TREES = [
    bq((bq((3, S), (7, S), (11, S), msm=2), M), (5, N)),                              # msm, MUST_NOT
    bq((bq((1, S), (2, S)), M), (bq((4, S), (P(A), N)), M)),
    DisjunctionMaxQuery([match(*C1), match(3, 5)], 0.0),                              # multi_match BEST_FIELDS
    bq((DisjunctionMaxQuery([match(*C1), match(3, 5)], 0.3), M), (PRICE, F)),
    P(A), P(B, 2), P(C8[:5]),                                                         # exact and sloppy phrases
    bq((match(*B), M), (BoostQuery(P(B), 2.0), S)),
    bq((MatchAllDocsQuery(), M), (bq((P(A), S), (9, S)), F)),                         # match-all and range leaves
    bq((bq((P(B[:2], 1), S), (3, S)), M), (PRICE, F)),
    P([B[2], B[1]]),                                                                  # every term occurs, never this phrase
]
SIX = [match(1, 2, 3, 4, 5, 6), bq((1, M), (3, S), (5, S), (7, S), (9, S), (11, S)), match(20, 40, 60, 80, 100, 120)]
WIDE_K = [match(3, 5), bq((7, S), (9, S), (P(A), S)), bq((2, M), (PRICE, F))]
NARROW = [match(1, 2), bq((3, M), (PRICE, F)), bq((4, S), (5, S), (6, S), msm=2), MatchAllDocsQuery()]

SORT1 = SortType(DBL, field_type="double", reverse=True)
SORT3 = [SortType(MV, selector="max", reverse=True), SortType(CAT, field_type="int", missing_last=True), SortType("docid")]
FILTER_Q = RangeQuery(0, 200_000, 900_000)
FILTER_SET = ValueSetFilter(DBL, (0.0, math.nan, -math.inf, 1.5), "double")


def collectors():
    return [
        TermsCollector(CAT, 6, field_type="int", nested=(("mx", MaxCollector(DBL, "double")), ("top", TopHitsCollector(3)),
                                                          ("s", SumCollector(0)), ("mn", MinCollector(DBL, "double"))),
                       order_by="s"),
        TermsCollector(CAT, 5, order_desc=False, field_type="int", nested=(("srt", TopHitsCollector(4, 1, SORT1)),)),
        MinCollector(DBL, "double"), MaxCollector(0), SumCollector(DBL, "double"),
        FilterCollector(FILTER_Q, (("set", FilterCollector(FILTER_SET, (("t", TermsCollector(CAT, 4, field_type="int", nested=(
            ("h", TopHitsCollector(5, 2, SORT3)),))), ("mx", MaxCollector(0))))),
                                   ("top", TopHitsCollector(4)))),
    ]


class Ref:
    def __init__(self, sh, oix, queries):
        self.sh, self.oix = sh, oix
        self.present, self.score = rtr.evaluate_all(sh, queries, oix)
        self._masks = {}

    def mask(self, f):
        if f not in self._masks:
            if isinstance(f, ValueSetFilter):
                self._masks[f] = far.value_set_mask(self.sh, f.column, f.sortable()).astype(bool)
            else:
                from nrtsearch_b200.search import compile_queries
                carr, _, qarr, _ = compile_queries([f])
                self._masks[f] = far.query_mask(self.oix, carr, qarr, 0)
        return self._masks[f]


def value_ok(g, want, what):
    v, bound = want
    if v is None:
        return
    if isinstance(v, float) and math.isnan(v):
        assert math.isnan(g), f"{what}: {g!r} vs NaN"
    elif bound == 0.0:
        assert g == v, f"{what}: {g!r} vs {v!r}"
    else:
        assert abs(g - v) <= bound, f"{what}: {g!r} vs {v!r} (bound {bound})"


def metric(R, c, sel):
    has = R.sh.column_has[c.column]
    d = np.nonzero(sel if has is None else sel & (np.asarray(has) != 0))[0]
    kind = "min" if isinstance(c, MinCollector) else "max" if isinstance(c, MaxCollector) else "sum"
    return nr.metric(kind, ar.as_doubles(np.asarray(R.sh.columns[c.column], np.int64)[d], VT[c.field_type]))


def check_hits(r, at, R, q, c, bucket, what):
    docs = np.nonzero(bucket)[0]
    fields = None if c.sort is None else sl.ref_fields(c.sort_fields())
    want, vals = shr.top_hits(R.sh, docs, R.score[q][docs], fields, c.top_hits, c.start_hit)
    m = len(want)
    assert r["counts"][at] == m and r["total_hits"][at] == len(docs), f"{what}: counts {r['counts'][at]} / {m}"
    assert r["docs"][at][:m].tolist() == want.tolist(), f"{what}: docs"
    if c.sort is None:
        assert np.array_equal(r["scores"][at][:m].view(np.uint32), R.score[q][want].view(np.uint32)), f"{what}: scores"
    else:
        assert np.array_equal(r["sort_values"][at][:m], vals), f"{what}: values"


def check(R, q, c, o, sel, what):
    """collector c's result o for query q over the docs `sel` its parent hands it"""
    if isinstance(c, TopHitsCollector):
        check_hits(o, q, R, q, c, sel, what)
    elif isinstance(c, (MinCollector, MaxCollector, SumCollector)):
        value_ok(float(o[q]), metric(R, c, sel), what)
    elif isinstance(c, FilterCollector):
        b = sel & R.mask(c.filter)
        assert o["doc_count"][q] == b.sum(), f"{what}: doc_count"
        for name, x in c.nested:
            check(R, q, x, o[name], b, f"{what}/{name}")
    else:
        specs = {name: ("min" if isinstance(x, MinCollector) else "max" if isinstance(x, MaxCollector) else "sum", x.column,
                        VT[x.field_type]) for name, x in c.nested if not isinstance(x, TopHitsCollector)}
        want = nr.terms_nested(R.sh, sel, c.column, c.size, c.order_desc, specs, c.order_by, R.score[q])
        n = want["n"]
        assert o["n"][q] == n and o["total_buckets"][q] == want["total_buckets"], f"{what}: buckets"
        assert o["keys"][q].tolist() == want["keys"].tolist() and o["counts"][q].tolist() == want["counts"].tolist(), f"{what}: keys"
        assert o["other_counts"][q] == want["other_counts"], f"{what}: other_counts"
        col, has = np.asarray(R.sh.columns[c.column]), R.sh.column_has[c.column]
        for name, x in c.nested:
            for i in range(n):
                if isinstance(x, TopHitsCollector):
                    b = sel & (col == o["keys"][q, i]) & (True if has is None else np.asarray(has) != 0)
                    check_hits(o["nested"][name], (q, i), R, q, x, b, f"{what}/{name} slot {i}")
                else:
                    value_ok(float(o["nested"][name][q, i]), want["nested"][name][i], f"{what}/{name} slot {i}")


def check_all(R, res, outs, colls, k, what):
    for q in range(len(res.counts)):
        for c, o in zip(colls, outs):
            check(R, q, c, o, R.present[q], f"{what} query {q} {type(c).__name__}")
        assert res.total_hits[q] == R.present[q].sum(), f"{what} query {q}: totalHits"


def same_page(a, b, what):
    assert np.array_equal(a.counts, b.counts), f"{what}: counts"
    assert np.array_equal(a.total_hits, b.total_hits), f"{what}: totalHits"
    assert np.array_equal(a.docs, b.docs), f"{what}: docs"
    assert np.array_equal(a.scores.view(np.uint32), b.scores.view(np.uint32)), f"{what}: scores"


def same_outs(a, b, what):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for key in a:
            same_outs(a[key], b[key], f"{what}/{key}")
    else:
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)), what


@pytest.fixture(scope="module")
def tree_run(corpus):
    sh, oix, g = corpus
    colls = collectors()
    res, outs = GpuIndexSearcher(g).search_tree_with_collectors(TREES, RelevanceCollector(10, INT_MAX), colls)
    return colls, res, outs, Ref(sh, oix, TREES)


def test_trees_and_phrases_against_the_references(tree_run):
    colls, res, outs, R = tree_run
    assert R.present.sum(axis=1)[-1] == 0 and (R.present.sum(axis=1)[:-1] > 0).all()
    check_all(R, res, outs, colls, 10, "trees")


def test_page_equals_search_tree(corpus, tree_run):
    _, _, g = corpus
    _, res, _, _ = tree_run
    same_page(res, GpuIndexSearcher(g).search_tree(TREES, RelevanceCollector(10, INT_MAX)), "trees")


@pytest.mark.parametrize("shape", ["six_terms", "top_k_1024"])
def test_wide_flat_batches(corpus, shape):
    sh, oix, g = corpus
    qs, k = (SIX, 10) if shape == "six_terms" else (WIDE_K, 1024)
    colls = collectors()
    s = GpuIndexSearcher(g)
    res, outs = s.search_tree_with_collectors(qs, RelevanceCollector(k, INT_MAX), colls)
    check_all(Ref(sh, oix, qs), res, outs, colls, k, shape)
    same_page(res, s.search_tree(qs, RelevanceCollector(k, INT_MAX)), shape)


def test_narrow_flat_batch_equals_search_with_collectors(corpus):
    _, _, g = corpus
    s = GpuIndexSearcher(g)
    a = s.search_tree_with_collectors(NARROW, RelevanceCollector(10, INT_MAX), collectors())
    b = s.search_with_collectors(NARROW, RelevanceCollector(10, INT_MAX), collectors())
    same_page(a[0], b[0], "narrow")
    for i, (x, y) in enumerate(zip(a[1], b[1])):
        same_outs(x, y, f"narrow collector {i}")


def test_three_leaves_equal_the_whole_image(corpus, leaves, tree_run):
    colls, res, outs, R = tree_run
    _, s = leaves
    lres, louts = s.search_tree_with_collectors(TREES, RelevanceCollector(10, INT_MAX), colls)
    same_page(lres, res, "leaves")
    check_all(R, lres, louts, colls, 10, "leaves")


def test_repeat_and_plain_search_after_collectors(corpus, tree_run):
    """a second identical call and a plain search_tree on the same pooled workspace see no state of the earlier call"""
    _, _, g = corpus
    colls, res, outs, _ = tree_run
    s = GpuIndexSearcher(g)
    again, again_outs = s.search_tree_with_collectors(TREES, RelevanceCollector(10, INT_MAX), colls)
    same_page(again, res, "repeat")
    for i, c in enumerate(colls):
        if isinstance(c, SumCollector):   # (a double sum's atomic additions may round in another order; the price sums are exact)
            continue
        same_outs(again_outs[i], outs[i], f"repeat collector {i}")
    plain = s.search_tree(TREES, RelevanceCollector(10, INT_MAX))
    s.search_tree_with_collectors(WIDE_K, RelevanceCollector(1024, INT_MAX), colls)
    same_page(s.search_tree(TREES, RelevanceCollector(10, INT_MAX)), plain, "plain after collectors")


def _raw_call(lib_fn, handle, qs, colls, orders_of, k=10):
    """the entry point called with sentinel-filled outputs; returns (status, outputs)"""
    carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(qs, phrase_table=True)
    fr = _FilteredRecords(nq, colls, orders_of)
    docs, scores = np.full((nq, k), -7, np.int32), np.full((nq, k), -7.0, np.float32)
    counts, total = np.full(nq, -7, np.int32), np.full(nq, -7, np.int64)
    rc = lib_fn(handle, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, k, 0, *fr.sorted_args, C.c_void_p(0),
                docs.ctypes.data, scores.ctypes.data, counts.ctypes.data, total.ctypes.data)
    return rc, (docs, scores, counts, total), fr.outs


def _untouched(outs, rc, what):
    assert rc != 0, what
    docs, scores, counts, total = outs
    assert (docs == -7).all() and (scores == -7.0).all() and (counts == -7).all() and (total == -7).all(), f"{what}: wrote output"


def test_refusals_write_nothing(gpu_ctx, corpus, leaves):
    from nrtsearch_b200 import _native
    sh, _, g = corpus
    ls, s = leaves
    lib = _native.gpu_lib()
    sorted_top = [TermsCollector(CAT, 3, field_type="int", nested=(("h", TopHitsCollector(3, 0, SORT1)),))]
    other = GpuIndex(gpu_ctx, sh.doc_range(0, 50_000))
    try:
        # an order made on another index
        rc, outs, _ = _raw_call(lib.nrtgpu_search_tree_aggs, g.handle, TREES, sorted_top,
                                lambda f: (C.c_void_p * 1)(other.sort_order(f).value))
        _untouched(outs, rc, "foreign order")
        rc, outs, _ = _raw_call(lib.nrtgpu_searcher_search_tree_aggs, s.handle, TREES, sorted_top,
                                lambda f: (C.c_void_p * len(ls))(*([other.sort_order(f).value] * len(ls))))
        _untouched(outs, rc, "searcher foreign order")
    finally:
        other.close()
    # a multi-valued column
    for fn, h in ((lib.nrtgpu_search_tree_aggs, g.handle), (lib.nrtgpu_searcher_search_tree_aggs, s.handle)):
        rc, outs, _ = _raw_call(fn, h, TREES, [TermsCollector(MV, 3)], None)
        _untouched(outs, rc, "multi-valued")
        assert rc == 3
    with pytest.raises(NrtGpuUnsupported):
        GpuIndexSearcher(g).search_tree_with_collectors(TREES, RelevanceCollector(10, INT_MAX), [TermsCollector(MV, 3)])
    # NULL arguments: no aggregations, a NULL searcher
    carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(TREES, phrase_table=True)
    docs = np.full((nq, 10), -7, np.int32)
    rc = lib.nrtgpu_search_tree_aggs(g.handle, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, 10, 0, None, 0, None, None, 0,
                                     None, None, None, None, 0, None, 0, C.c_void_p(0), docs.ctypes.data, None, None, None)
    assert rc == 1 and (docs == -7).all()
    rc = lib.nrtgpu_searcher_search_tree_aggs(None, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, 10, 0, None, 0, None, None,
                                              0, None, None, None, None, 0, None, 0, C.c_void_p(0), docs.ctypes.data, None, None, None)
    assert rc == 1 and (docs == -7).all()
    with pytest.raises(NrtGpuError):
        GpuIndexSearcher(g).search_tree_with_collectors(TREES, RelevanceCollector(10, INT_MAX), [])
