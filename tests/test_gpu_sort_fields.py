"""Sort on several fields on the GPU path (nrtgpu_sort_order / nrtgpu_search_sorted_fields): multi-key Sorts of numeric columns
and doc ids, MIN / MAX selectors on a multi-valued column, a leading score, searchAfter, against the exhaustive reference
(tests/sort_fields_reference.py, on the oracle's matching and scoring), bit-exact on docs, every FieldDoc value, counts and totals."""
import copy
import ctypes as C

import numpy as np
import pytest

import sort_fields_reference as ref
from nrtsearch_b200 import _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, FieldDoc, GpuIndex, GpuIndexSearcher, MatchAllDocsQuery, NrtGpuUnsupported, Occur, RangeQuery, ScoreDoc, SortFieldCollector, SortType, TermQuery,
                                   compile_queries, float_to_sortable_int)

pytestmark = pytest.mark.gpu

N_DOCS, VOCAB, DOC_BASE = 600_000, 8_000, 3_000   # two probe slices; results carry doc_base + local


def make_shard():
    sh = ix.synth_text_shard(N_DOCS, VOCAB, min_len=6, poisson_mean=30.0)
    sh.doc_base = DOC_BASE
    rng = np.random.default_rng(29)
    n = N_DOCS
    c_int = rng.integers(0, 8, n).astype(np.int64)                                           # low cardinality: multi-key ties
    c_float = np.array([float_to_sortable_int(x) for x in (-2.5, -0.5, 0.0, 1.25, 3.0, 7.5)], np.int64)[rng.integers(0, 6, n)]
    c_long = rng.integers(-4, 4, n).astype(np.int64) * (2**60)
    cnt = rng.integers(0, 4, n)                                                               # 0..3 values per doc
    off = np.zeros(n + 1, np.int64)
    np.cumsum(cnt, out=off[1:])
    vals = rng.integers(-20, 20, int(off[-1])).astype(np.int64)
    vals = vals[np.lexsort((vals, np.repeat(np.arange(n), cnt)))]                             # ascending within a doc
    sh.columns = [c_int, c_float, c_long, vals]
    sh.column_has = [(rng.random(n) < 0.85).astype(np.uint8), (rng.random(n) < 0.8).astype(np.uint8),
                     (rng.random(n) < 0.9).astype(np.uint8), None]
    sh.column_offsets = [None, None, None, off]
    sh.live_docs = (rng.random(n) < 0.92).astype(np.uint8)
    return sh


def make_queries():
    terms = ix.synth_query_terms(12, 3, VOCAB, seed=77, log10_lo=0.5, log10_hi=3.3)
    qs = []
    for i, t in enumerate(terms):
        a, b, c = (int(x) for x in t)
        kind = i % 6
        if kind == 0:
            qs.append(BooleanQuery().add(TermQuery(a), Occur.SHOULD).add(TermQuery(b), Occur.SHOULD).add(TermQuery(c), Occur.SHOULD))
        elif kind == 1:
            qs.append(BooleanQuery().add(TermQuery(a), Occur.MUST).add(RangeQuery(0, 2, 5), Occur.FILTER))
        elif kind == 2:
            qs.append(BooleanQuery().add(TermQuery(a), Occur.SHOULD).add(TermQuery(b), Occur.SHOULD).add(TermQuery(c), Occur.MUST_NOT))
        elif kind == 3:
            qs.append(MatchAllDocsQuery())
        elif kind == 4:
            qs.append(RangeQuery(0, 1, 3))
        else:
            qs.append(BooleanQuery())   # matches nothing
    return qs


SPECS = {
    "int,float": [SortType(0, field_type="int"), SortType(1, field_type="float")],
    "int-desc,long-missing-last": [SortType(0, True, field_type="int"), SortType(2, missing_last=True, field_type="long")],
    "float,docid-desc": [SortType(1, field_type="float"), SortType("docid", True)],
    "int,docid,long": [SortType(0, field_type="int"), SortType("docid"), SortType(2, field_type="long")],
    "multi-min,int": [SortType(3, field_type="int"), SortType(0, field_type="int")],
    "multi-max-desc": [SortType(3, True, selector="max", field_type="int")],
    "score": [SortType("score")],
    "score-reverse": [SortType("score", True)],
    "score,int-desc": [SortType("score"), SortType(0, True, field_type="int")],
    "score,multi-max,long": [SortType("score"), SortType(3, selector="max", field_type="int"), SortType(2, field_type="long")],
}


def ref_fields(spec):
    return [tuple(getattr(f.c_field(), n) for n in ("kind", "column", "reverse", "selector", "missing_value")) for f in spec]


def want(sh, qs, k, spec, after=None):
    sd = None if after is None else [ScoreDoc(a.doc, 0.0) for a in after]
    carr, ncl, qarr, nq = compile_queries(qs, sd)
    av = None if after is None else [list(a.values) for a in after]
    return ref.search_sorted_fields(sh, carr, ncl, qarr, nq, k, ref_fields(spec), av)


def assert_equal(res, w, k, what=""):
    wd, wv, wc, wt = w
    assert np.array_equal(res.counts, np.minimum(wc, k)), what
    assert np.array_equal(res.total_hits, wt) and not res.relation.any(), what
    for q in range(len(res.counts)):
        n = res.counts[q]
        assert np.array_equal(res.docs[q, :n], wd[q, :n]), (what, q, res.docs[q, :6], wd[q, :6])
        assert np.array_equal(res.sort_values[q, :n], wv[q, :n]), (what, q)


@pytest.fixture(scope="module")
def setup(gpu_ctx):
    sh = make_shard()
    gix = GpuIndex(gpu_ctx, sh)
    yield sh, make_queries(), gix
    gix.close()


@pytest.mark.parametrize("name", list(SPECS))
def test_specs_equal_reference(setup, name):
    sh, qs, gix = setup
    spec = SPECS[name]
    w = want(sh, qs, 512, spec)
    s = GpuIndexSearcher(gix)
    for k in (1, 40, 512):
        res = s.search_sorted(qs, SortFieldCollector(k, spec))
        assert res.sort_values.shape == (len(qs), k, len(spec))
        assert_equal(res, w, k, f"{name} k={k}")


@pytest.mark.parametrize("name", ["int,float", "multi-max-desc", "score", "score,int-desc", "int,docid,long"])
def test_search_after_pages(setup, name):
    sh, qs, gix = setup
    spec, k = SPECS[name], 40
    s = GpuIndexSearcher(gix)
    p1 = s.search_sorted(qs, SortFieldCollector(k, spec))
    sel = [q for q in range(len(qs)) if p1.counts[q] == k]
    after = [FieldDoc(int(p1.docs[q, k - 1]), values=tuple(int(x) for x in p1.sort_values[q, k - 1])) for q in sel]
    sub = [qs[q] for q in sel]
    p2 = s.search_sorted(sub, SortFieldCollector(k, spec), search_after=after)
    assert_equal(p2, want(sh, sub, k, spec, after), k, name)
    full = s.search_sorted(sub, SortFieldCollector(2 * k, spec))
    for i, q in enumerate(sel):   # no gap, no overlap
        assert np.array_equal(np.concatenate([p1.docs[q, :k], p2.docs[i, :p2.counts[i]]]), full.docs[i, :k + p2.counts[i]])


@pytest.mark.parametrize("name", ["int,float", "float,docid-desc", "score,int-desc", "multi-min,int"])
def test_after_values_absent_from_the_index_and_after_doc_outside_the_leaf(setup, name):
    sh, qs, gix = setup
    spec, k = SPECS[name], 40
    absent = {0: [-1, 3, 100], 1: [float_to_sortable_int(x) for x in (-9.0, 0.75, 50.0)], 3: [-30, 4, 30]}
    rng = np.random.default_rng(5)
    after, sub = [], []
    for i, q in enumerate(qs):
        vals = []
        for f in spec:
            if f.field == "score":
                vals.append(int(np.float32(rng.choice([0.0, 2.5, 6.0, 40.0])).view(np.uint32)))
            elif f.field == "docid":
                vals.append(int(rng.choice([0, DOC_BASE + N_DOCS // 3, DOC_BASE + N_DOCS + 9])))
            else:
                vals.append(int(rng.choice(absent[f.field])))
        for adoc in (0, DOC_BASE + N_DOCS // 2, DOC_BASE + N_DOCS + 9):   # below, inside and above the leaf
            after.append(FieldDoc(adoc, values=tuple(vals)))
            sub.append(q)
    res = GpuIndexSearcher(gix).search_sorted(sub, SortFieldCollector(k, spec), search_after=after)
    assert_equal(res, want(sh, sub, k, spec, after), k, name)


def test_one_field_order_equals_the_single_field_path(setup):
    sh, qs, gix = setup
    s = GpuIndexSearcher(gix)
    for st in (SortType(0, field_type="int"), SortType(1, True, True, "float"), SortType(2, False, True, "long"), SortType("docid", True)):
        one = s.search_sorted(qs, SortFieldCollector(40, st))
        many = s.search_sorted(qs, SortFieldCollector(40, [st]))
        assert np.array_equal(one.counts, many.counts) and np.array_equal(one.total_hits, many.total_hits)
        assert np.array_equal(one.docs, many.docs) and np.array_equal(one.sort_values, many.sort_values[:, :, 0])


def test_order_stays_valid_after_deletes_and_stats_refresh(gpu_ctx):
    sh = make_shard()
    qs = make_queries()
    gix = GpuIndex(gpu_ctx, sh)
    try:
        s = GpuIndexSearcher(gix)
        fields_spec, score_spec = SPECS["int-desc,long-missing-last"], SPECS["score,multi-max,long"]
        assert_equal(s.search_sorted(qs, SortFieldCollector(40, fields_spec)), want(sh, qs, 40, fields_spec), 40, "before")
        assert_equal(s.search_sorted(qs, SortFieldCollector(40, score_spec)), want(sh, qs, 40, score_spec), 40, "before")
        n_orders = len(gix._orders)
        sh2 = copy.copy(sh)
        sh2.live_docs = (np.random.default_rng(8).random(N_DOCS) < 0.7).astype(np.uint8)
        gix.set_live_docs(sh2.live_docs)
        assert_equal(s.search_sorted(qs, SortFieldCollector(40, fields_spec)), want(sh2, qs, 40, fields_spec), 40, "deletes")
        sh3 = copy.copy(sh2)
        sh3.fields = [ix.TextField(f.norms, f.doc_count * 3, f.sum_total_term_freq * 2, f.k1, f.b) for f in sh2.fields]
        sh3.term_df = np.asarray(sh2.term_df if sh2.term_df is not None else np.diff(sh2.term_off), np.int64) * 2 + 1
        gix.update_stats(sh3.term_df, [f.doc_count for f in sh3.fields], [f.sum_total_term_freq for f in sh3.fields])
        assert_equal(s.search_sorted(qs, SortFieldCollector(40, score_spec)), want(sh3, qs, 40, score_spec), 40, "stats")
        assert len(gix._orders) == n_orders   # the cached orders were reused
        lib = _native.gpu_lib()
        assert all(lib.nrtgpu_sort_order_device_bytes(h) == 8 * N_DOCS for h in gix._orders.values())
    finally:
        gix.close()


def test_limits(setup):
    sh, qs, gix = setup
    spec = SPECS["score,int-desc"]
    s = GpuIndexSearcher(gix)
    res = s.search_sorted(qs, SortFieldCollector(40, spec, terminate_after=100))
    assert res.terminated_early[3] == 1 and res.relation[3] == 1   # match-all: far more than 100 matches
    lib = _native.gpu_lib()
    order = gix.sort_order(spec)
    carr, ncl, qarr, nq = compile_queries(qs)
    k = 40
    docs, vals = np.zeros((nq, k), np.int32), np.zeros((nq, k, 2), np.int64)
    cnt, tot, rel, to, te = (np.zeros(nq, t) for t in (np.int32, np.int64, np.uint8, np.uint8, np.uint8))
    lim = _native.SearchLimits(0.5, 1.0, 0, 0, 0)   # the request spent its budget before the call
    rc = lib.nrtgpu_search_sorted_fields(gix.handle, order, carr, ncl, qarr, nq, k, 0, None, C.byref(lim), None, docs.ctypes.data,
                                         vals.ctypes.data, cnt.ctypes.data, tot.ctypes.data, rel.ctypes.data, to.ctypes.data,
                                         te.ctypes.data)
    assert rc == 0
    assert to[3] == 1 and rel[3] == 1


def test_refusals(setup, gpu_ctx):
    sh, qs, gix = setup
    lib = _native.gpu_lib()
    F = _native.SortField

    def create(fields, index=gix):
        arr = (F * max(len(fields), 1))(*fields)
        h = C.c_void_p()
        rc = lib.nrtgpu_sort_order_create(index.handle, arr, len(fields), None, C.byref(h))
        if rc == 0:
            lib.nrtgpu_sort_order_close(h)
        return rc

    INVALID, UNSUPPORTED = 1, 3
    assert create([]) == INVALID
    assert create([F(7, 0, 0, 0, 0)]) == INVALID                   # bad kind
    assert create([F(1, 0, 0, 2, 0)]) == INVALID                   # bad selector
    assert create([F(1, 99, 0, 0, 0)]) == INVALID                  # column out of range
    assert create([F(2, 0, 0, 0, 0)] * 9) == UNSUPPORTED
    assert create([F(1, 0, 0, 0, 0), F(3, 0, 0, 0, 0)]) == UNSUPPORTED   # score after a column
    assert create([F(3, 0, 1, 0, 0), F(1, 3, 0, 1, 0), F(2, 0, 0, 0, 0), F(1, 0, 0, 0, 0)]) == 0   # fields after a doc id are accepted
    s = GpuIndexSearcher(gix)
    spec = SPECS["int,float"]
    # an order made on another index
    other = GpuIndex(gpu_ctx, ix.synth_text_shard(10_000, 500))
    try:
        foreign = other.sort_order([SortType("docid")])
        carr, ncl, qarr, nq = compile_queries(qs[:2])
        out = [np.zeros(64, np.int64) for _ in range(7)]
        rc = lib.nrtgpu_search_sorted_fields(gix.handle, foreign, carr, ncl, qarr, nq, 4, 0, None, None, None,
                                             *[o.ctypes.data for o in out])
        assert rc == INVALID
    finally:
        other.close()
    # searchAfter without after values
    carr, ncl, qarr, nq = compile_queries(qs[:2], [ScoreDoc(DOC_BASE + 5, 0.0)] * 2)
    out = [np.zeros(64, np.int64) for _ in range(7)]
    rc = lib.nrtgpu_search_sorted_fields(gix.handle, gix.sort_order(spec), carr, ncl, qarr, nq, 4, 0, None, None, None,
                                         *[o.ctypes.data for o in out])
    assert rc == INVALID
    # wide batches
    t = [int(x) for x in ix.synth_query_terms(1, 5, VOCAB, seed=3)[0]]
    five = BooleanQuery()
    for x in t:
        five.add(TermQuery(x), Occur.SHOULD)
    with pytest.raises(NrtGpuUnsupported):
        s.search_sorted([five], SortFieldCollector(10, spec))
    with pytest.raises(NrtGpuUnsupported):
        s.search_sorted(qs[:2], SortFieldCollector(513, spec))
    with pytest.raises(ValueError):
        s.search_sorted(qs[:2], SortFieldCollector(10, [SortType(0, selector="median")]))
