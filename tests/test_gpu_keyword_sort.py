"""Sort by keyword fields on the GPU path (NRTGPU_SORT_KEYWORD in nrtgpu_sort_order; SortType(field_type="keyword")): SORTED
and SORTED_SET string sort fields with every selector and missing rule, alone and mixed with numeric, doc id and leading
score fields, searchAfter by term, three doc-range leaves with dictionaries of their own, and sorted top hits, against
tests/keyword_sort_reference.py (on the oracle's matching and scoring), bit-exact on docs, every FieldDoc value, counts,
totals and flags.

The shard has two probe slices and deletes. Its keyword columns: SORTED over a dictionary with the empty string, the
prefixes a < a\\x00 < ab and multi-byte UTF-8 (a 4-byte character among them), 12 % of docs without a value, later docs
drawing from more terms; SORTED_SET of 0-5 terms per doc; a column of one term; a column without values."""
import copy
import ctypes as C

import numpy as np
import pytest

import keyword_sort_reference as ref
from nrtsearch_b200 import NrtGpuError, _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200.index import KeywordColumn
from nrtsearch_b200.search import (BooleanQuery, FieldDoc, FilterCollector, GpuIndex, GpuIndexSearcher, GpuLeafSearcher,
                                   MatchAllDocsQuery, Occur, RangeQuery, RelevanceCollector, ScoreDoc,
                                   SortFieldCollector, SortType, TermQuery, TermsCollector, TopHitsCollector, compile_queries)

pytestmark = pytest.mark.gpu

N_DOCS, VOCAB, DOC_BASE = 400_000, 8_000, 2_000
INT = 0                                   # numeric column: 0..7, 85 % with a value
KW, KW_SET, KW_ONE, KW_NONE = 0, 1, 2, 3  # keyword columns
CUTS = [0, 120_001, 290_000]
SPECIAL = ["", "a", "a\x00", "ab", "b", "café", "cafe", "Zürich", "\U0001f355", "ÿ", "z"]


def keyword_columns(n, rng):
    words = SPECIAL + [f"w{i:03d}" for i in range(300)]
    lim = 40 + (np.arange(n) * (len(words) - 40)) // n   # later docs draw from more terms: the leaves' dictionaries differ
    one = [None if rng.random() < 0.12 else words[int(rng.integers(0, lim[d]))] for d in range(n)]
    per = rng.integers(0, 6, n)
    sets = [[words[int(x)] for x in rng.integers(0, lim[d], p)] for d, p in enumerate(per)]
    solo = [None if d % 3 else "solo" for d in range(n)]
    return [KeywordColumn.from_values(one, False), KeywordColumn.from_values(sets, True), KeywordColumn.from_values(solo, False),
            KeywordColumn.from_values([None] * n, False)]


def make_shard():
    sh = ix.synth_text_shard(N_DOCS, VOCAB, min_len=6, poisson_mean=30.0)
    sh.doc_base = DOC_BASE
    rng = np.random.default_rng(0x50F7)
    sh.columns = [rng.integers(0, 8, N_DOCS).astype(np.int64)]
    sh.column_has = [(rng.random(N_DOCS) < 0.85).astype(np.uint8)]
    sh.column_offsets = [None]
    sh.keyword_columns = keyword_columns(N_DOCS, rng)
    sh.live_docs = (rng.random(N_DOCS) < 0.92).astype(np.uint8)
    return sh


def make_queries():
    terms = ix.synth_query_terms(6, 3, VOCAB, seed=71, log10_lo=0.5, log10_hi=3.3)
    qs = []
    for i, t in enumerate(terms):
        a, b, c = (int(x) for x in t)
        kind = i % 6
        if kind == 0:
            qs.append(BooleanQuery().add(TermQuery(a), Occur.SHOULD).add(TermQuery(b), Occur.SHOULD).add(TermQuery(c), Occur.SHOULD))
        elif kind == 1:
            qs.append(BooleanQuery().add(TermQuery(a), Occur.MUST).add(RangeQuery(INT, 2, 5), Occur.FILTER))
        elif kind == 2:
            qs.append(BooleanQuery().add(TermQuery(a), Occur.SHOULD).add(TermQuery(b), Occur.SHOULD).add(TermQuery(c), Occur.MUST_NOT))
        elif kind == 3:
            qs.append(MatchAllDocsQuery())
        elif kind == 4:
            qs.append(RangeQuery(INT, 1, 3))
        else:
            qs.append(BooleanQuery())   # matches nothing
    return qs


def K(col=KW, reverse=False, missing_last=False, selector="min"):
    return SortType(col, reverse, missing_last, "keyword", selector)


I_ASC, I_DESC = SortType(INT, field_type="int"), SortType(INT, True, field_type="int")
SPECS = {
    "kw": [K()], "kw-desc": [K(reverse=True)], "kw-missing-last": [K(missing_last=True)],
    "kw-desc-missing-last": [K(reverse=True, missing_last=True)],
    **{f"set-{sel}{'-desc' if r else ''}": [K(KW_SET, r, selector=sel)] for sel in ("min", "max", "middle_min", "middle_max")
       for r in (False, True)},
    "kw,int": [K(), I_ASC], "int-desc,kw": [I_DESC, K()], "score,kw": [SortType("score"), K(missing_last=True)],
    "kw,docid": [K(reverse=True), SortType("docid")], "kw,kw_set-max": [K(), K(KW_SET, selector="max")],
    "one-term,none,int": [K(KW_ONE, missing_last=True), K(KW_NONE, True), I_DESC],
}


def ref_fields(spec):
    return [tuple(getattr(f.c_field(), n) for n in ("kind", "column", "reverse", "selector", "missing_value")) for f in spec]


def enc(v):
    """a GPU FieldDoc value in the reference's terms (str -> UTF-8 bytes)"""
    return v.encode("utf-8") if isinstance(v, str) else v


def ref_after(spec, a):
    return [enc(x) for x in (a.values if a.values is not None else (a.value,))]


def want(sh, qs, k, spec, after=None, restrict=None):
    sd = None if after is None else [ScoreDoc(a.doc, 0.0) for a in after]
    carr, ncl, qarr, nq = compile_queries(qs, sd)
    av = None if after is None else [ref_after(spec, a) for a in after]
    return ref.search(sh, carr, ncl, qarr, nq, k, ref_fields(spec), av, restrict=restrict)


def rows(vals, n):
    """the first n FieldDoc tuples of one query, keyword entries as bytes"""
    v = np.asarray(vals)
    v = v.reshape(v.shape[0], -1)
    return [tuple(enc(x) for x in v[i]) for i in range(n)]


def assert_equal(res, w, k, what=""):
    wd, wv, wc, wt = w
    assert np.array_equal(res.counts, np.minimum(wc, k)), what
    assert np.array_equal(res.total_hits, wt) and not res.relation.any(), what
    for q in range(len(res.counts)):
        n = res.counts[q]
        assert np.array_equal(res.docs[q, :n], wd[q, :n]), (what, q, res.docs[q, :6], wd[q, :6])
        assert rows(res.sort_values[q], n) == rows(wv[q], n), (what, q)


@pytest.fixture(scope="module")
def setup(gpu_ctx):
    sh = make_shard()
    gix = GpuIndex(gpu_ctx, sh)
    yield sh, make_queries(), gix
    gix.close()


@pytest.fixture(scope="module")
def leaves(gpu_ctx, setup):
    sh = setup[0]
    cuts = CUTS + [N_DOCS]
    subs = [sh.doc_range(a, b) for a, b in zip(cuts, cuts[1:])]
    assert len({len(s.keyword_columns[KW].terms) for s in subs}) == 3   # three different dictionaries
    ls = [GpuIndex(gpu_ctx, s) for s in subs]
    s = GpuLeafSearcher(gpu_ctx, ls)
    yield ls, s
    s.close()
    for g in ls:
        g.close()


@pytest.mark.parametrize("name", list(SPECS))
def test_specs_equal_reference(setup, name):
    sh, qs, gix = setup
    spec = SPECS[name]
    w = want(sh, qs, 512, spec)
    s = GpuIndexSearcher(gix)
    for k in (1, 40, 512):
        res = s.search_sorted(qs, SortFieldCollector(k, spec))
        assert res.sort_values.dtype == object and res.sort_values.shape == (len(qs), k, len(spec))
        assert_equal(res, w, k, f"{name} k={k}")


def test_one_keyword_sort_type_is_a_one_field_order(setup):
    sh, qs, gix = setup
    s = GpuIndexSearcher(gix)
    one = s.search_sorted(qs, SortFieldCollector(40, K(reverse=True)))
    many = s.search_sorted(qs, SortFieldCollector(40, [K(reverse=True)]))
    assert one.sort_values.shape == (len(qs), 40)
    assert np.array_equal(one.docs, many.docs) and list(one.sort_values.reshape(-1)) == list(many.sort_values[:, :, 0].reshape(-1))
    assert all(x is None or isinstance(x, str) for x in one.sort_values.reshape(-1))
    nums = s.search_sorted(qs, SortFieldCollector(40, [I_DESC, SortType("docid")]))
    assert nums.sort_values.dtype == np.int64   # all-numeric Sorts keep int64 values


@pytest.mark.parametrize("name", ["kw", "kw-desc-missing-last", "set-middle_max-desc", "int-desc,kw", "score,kw", "kw,kw_set-max"])
def test_page_walk(setup, name):
    sh, qs, gix = setup
    spec, k, pages = SPECS[name], 37, 5
    s = GpuIndexSearcher(gix)
    full = s.search_sorted(qs, SortFieldCollector(k * pages, spec))
    got = [[] for _ in qs]
    after, prev = None, [FieldDoc(0, values=tuple(None if f.keyword else 0 for f in spec)) for _ in qs]
    for _ in range(pages):
        res = s.search_sorted(qs, SortFieldCollector(k, spec), search_after=after)
        for q in range(len(qs)):
            n = int(res.counts[q])
            got[q] += res.docs[q, :n].tolist()
            if n:   # the last hit's FieldDoc, values as str / None / int (an exhausted query keeps its last one)
                prev[q] = FieldDoc(int(res.docs[q, n - 1]), values=tuple(res.sort_values[q, n - 1]))
        after = list(prev)
    for q in range(len(qs)):
        n = min(full.counts[q], len(got[q]))
        assert got[q][:n] == full.docs[q, :n].tolist(), (name, q)
        assert len(got[q]) == full.counts[q] or full.counts[q] == k * pages, (name, q)


@pytest.mark.parametrize("name", ["kw", "kw-desc", "kw-missing-last", "kw-desc-missing-last", "set-middle_min", "kw,int"])
def test_synthetic_after_values(setup, name):
    sh, qs, gix = setup
    spec, k = SPECS[name], 40
    terms = [None, "", "\x00", "a\x00\x00", "a\x00", "cafe\x00", "w150", "w150a", "\U0010ffff"]   # held, absent, null, ""
    after, sub = [], []
    for i, q in enumerate(qs[:3] + qs[3:4]):   # (the match-all query with three of the terms: the reference's cost)
        for j, t in enumerate(terms if i < 3 else terms[::4]):
            vals = tuple(t if f.keyword else (3 if j % 2 else 0) for f in spec)
            for adoc in (0, DOC_BASE + N_DOCS // 2, DOC_BASE + N_DOCS + 9):
                after.append(FieldDoc(adoc, values=vals))
                sub.append(q)
    res = GpuIndexSearcher(gix).search_sorted(sub, SortFieldCollector(k, spec), search_after=after)
    assert_equal(res, want(sh, sub, k, spec, after), k, name)


@pytest.mark.parametrize("name", ["kw", "kw-desc-missing-last", "set-middle_min-desc", "int-desc,kw", "score,kw", "kw,kw_set-max"])
def test_leaves_equal_the_whole_image(setup, leaves, name):
    sh, qs, gix = setup
    _, s = leaves
    spec, k = SPECS[name], 60
    whole = GpuIndexSearcher(gix).search_sorted(qs, SortFieldCollector(k, spec))
    res = s.search_sorted(qs, SortFieldCollector(k, spec))
    assert np.array_equal(res.counts, whole.counts) and np.array_equal(res.total_hits, whole.total_hits)
    for q in range(len(qs)):
        n = res.counts[q]
        assert np.array_equal(res.docs[q, :n], whole.docs[q, :n]), (name, q)
        assert rows(res.sort_values[q], n) == rows(whole.sort_values[q], n), (name, q)
    # searchAfter by reader-wide terms: held by some leaves only ("w299" only by the last), by none, and null
    after, sub = [], []
    for q in range(len(qs)):
        for t in (None, "", "w010", "w299", "w2999", "a\x00\x01", "\U0010ffff"):
            after.append(FieldDoc(DOC_BASE + 150_000, values=tuple(t if f.keyword else 2 for f in spec)))
            sub.append(qs[q])
    res = s.search_sorted(sub, SortFieldCollector(k, spec), search_after=after)
    assert_equal(res, want(sh, sub, k, spec, after), k, name)
    img = GpuIndexSearcher(gix).search_sorted(sub, SortFieldCollector(k, spec), search_after=after)
    assert np.array_equal(img.docs, res.docs)


HIT_SORT = [K(KW_SET, True, True, "middle_max"), K(), I_ASC]


def hits_rows(h, idx, n):
    return h["docs"][idx][:n].tolist(), rows(h["sort_values"][idx], n)


def test_sorted_top_hits(setup, leaves):
    sh, qs, gix = setup
    ls, s = leaves
    qs = qs[:5]
    th = TopHitsCollector(7, 0, HIT_SORT)
    filt = RangeQuery(INT, 2, 6)
    coll = [th, TermsCollector(INT, 4, nested=(("top", th),)), TermsCollector(KW_SET, 3, field_type="keyword", nested=(("top", th),)),
            FilterCollector(filt, nested=(("top", th),))]
    img = GpuIndexSearcher(gix).search_with_collectors(qs, RelevanceCollector(10), coll)[1]
    lv = s.search_with_collectors(qs, RelevanceCollector(10), coll)[1]
    # top level and under the filter: the sorted search of the same queries, cut to the filter's docs
    col, has = sh.columns[INT], sh.column_has[INT] != 0
    for out in (img, lv):
        for got, cut in ((out[0], None), (out[3]["top"], has & (col >= 2) & (col <= 6))):
            w = want(sh, qs, 7, HIT_SORT, restrict=cut)
            for q in range(len(qs)):
                n = int(got["counts"][q])
                assert n == min(w[2][q], 7)
                assert hits_rows(got, q, n) == (w[0][q, :n].tolist(), rows(w[1][q], n)), q
                assert all(x is None or isinstance(x, str) for x in got["sort_values"][q][:n, :2].reshape(-1))
        # under a numeric terms bucket: the sorted search of the query filtered to the bucket's value
        t = out[1]
        for q in range(len(qs)):
            for b in range(int(t["n"][q])):
                v = int(t["keys"][q, b])
                w = want(sh, [qs[q]], 7, HIT_SORT, restrict=has & (col == v))
                n = int(t["nested"]["top"]["counts"][q, b])
                assert hits_rows(t["nested"]["top"], (q, b), n) == (w[0][0, :n].tolist(), rows(w[1][0], n)), (q, b)
    # under a keyword terms bucket: leaves with dictionaries of their own give the image's hits and terms
    a, b2 = img[2], lv[2]
    assert list(a["keys"].reshape(-1)) == list(b2["keys"].reshape(-1))
    assert np.array_equal(a["nested"]["top"]["docs"], b2["nested"]["top"]["docs"])
    assert list(a["nested"]["top"]["sort_values"].reshape(-1)) == list(b2["nested"]["top"]["sort_values"].reshape(-1))


def test_sorted_top_hits_on_the_window_engine(setup, leaves):
    sh, qs, gix = setup
    t = [int(x) for x in ix.synth_query_terms(2, 2, VOCAB, seed=9, log10_lo=1.0, log10_hi=3.0).reshape(-1)]
    nested = [BooleanQuery().add(BooleanQuery().add(TermQuery(t[0]), Occur.SHOULD).add(TermQuery(t[1]), Occur.SHOULD), Occur.MUST)]
    flat = [BooleanQuery().add(TermQuery(t[0]), Occur.SHOULD).add(TermQuery(t[1]), Occur.SHOULD)]
    th = TopHitsCollector(9, 2, HIT_SORT)
    for searcher in (GpuIndexSearcher(gix), leaves[1]):
        tree = searcher.search_tree_with_collectors(nested, RelevanceCollector(10), [th])[1][0]
        w = want(sh, flat, 9, HIT_SORT)
        n = int(tree["counts"][0])
        assert n == max(min(w[2][0], 9) - 2, 0)
        assert hits_rows(tree, 0, n) == (w[0][0, 2:2 + n].tolist(), rows(w[1][0, 2:], n))


def known_shard(n, kw, ints=None):
    sh = ix.synth_text_shard(n, 20, min_len=2, poisson_mean=2.0)
    sh.columns = [np.array([0 if v is None else v for v in (ints or [None] * n)], np.int64)]
    sh.column_has = [np.array([v is not None for v in (ints or [None] * n)], np.uint8)]
    sh.column_offsets = [None]
    sh.keyword_columns = [KeywordColumn.from_values(kw, False)]
    return sh


def test_sort_field_test_known_answers(gpu_ctx):
    INT_MIN = -(2**31)
    sh = known_shard(10, [None if i < 5 else str(9 - i) for i in range(10)], [i if i < 5 else None for i in range(10)])
    g = GpuIndex(gpu_ctx, sh)
    try:
        s = GpuIndexSearcher(g)
        for ir, sr, ids, strs in ((False, False, [9, 8, 7, 6, 5, 0, 1, 2, 3, 4], ["0", "1", "2", "3", "4"] + [None] * 5),
                                  (True, False, [4, 3, 2, 1, 0, 9, 8, 7, 6, 5], [None] * 5 + ["0", "1", "2", "3", "4"]),
                                  (False, True, [5, 6, 7, 8, 9, 0, 1, 2, 3, 4], ["4", "3", "2", "1", "0"] + [None] * 5),
                                  (True, True, [4, 3, 2, 1, 0, 5, 6, 7, 8, 9], [None] * 5 + ["4", "3", "2", "1", "0"])):
            r = s.search_sorted([MatchAllDocsQuery()], SortFieldCollector(10, [SortType(0, ir, field_type="int"), K(0, sr)]))
            assert r.docs[0].tolist() == ids and list(r.sort_values[0, :, 1]) == strs
        spec = [K(0), SortType(0, True, field_type="int")]
        r = s.search_sorted([MatchAllDocsQuery()], SortFieldCollector(3, spec))
        assert r.docs[0].tolist() == [4, 3, 2] and [tuple(x) for x in r.sort_values[0]] == [(None, 4), (None, 3), (None, 2)]
        r = s.search_sorted([MatchAllDocsQuery()], SortFieldCollector(3, spec), search_after=[FieldDoc(2, values=(None, 2))])
        assert r.docs[0].tolist() == [1, 0, 9] and [tuple(x) for x in r.sort_values[0]] == [(None, 1), (None, 0), ("0", INT_MIN)]
    finally:
        g.close()
    whole = known_shard(100, [str(i) for i in range(100)])
    ls = [GpuIndex(gpu_ctx, whole.doc_range(10 * i, 10 * i + 10)) for i in range(10)]
    ls_s = GpuLeafSearcher(gpu_ctx, ls)
    try:
        r = ls_s.search_sorted([MatchAllDocsQuery()], SortFieldCollector(5, K(0)))
        assert list(r.sort_values[0]) == ["0", "1", "10", "11", "12"] and r.docs[0].tolist() == [0, 1, 10, 11, 12]
        r = ls_s.search_sorted([MatchAllDocsQuery()], SortFieldCollector(5, K(0)), search_after=[FieldDoc(0, "1")])
        assert list(r.sort_values[0]) == ["1", "10", "11", "12", "13"]
    finally:
        ls_s.close()
        for g in ls:
            g.close()


def test_order_reused_after_deletes_and_limits(gpu_ctx, setup):
    sh0, qs, _ = setup
    sh = copy.copy(sh0)
    gix = GpuIndex(gpu_ctx, sh)
    try:
        s = GpuIndexSearcher(gix)
        spec = SPECS["kw,int"]
        assert_equal(s.search_sorted(qs, SortFieldCollector(40, spec)), want(sh, qs, 40, spec), 40, "before")
        n_orders = len(gix._orders)
        sh2 = copy.copy(sh)
        sh2.live_docs = (np.random.default_rng(8).random(N_DOCS) < 0.7).astype(np.uint8)
        gix.set_live_docs(sh2.live_docs)
        assert_equal(s.search_sorted(qs, SortFieldCollector(40, spec)), want(sh2, qs, 40, spec), 40, "deletes")
        assert len(gix._orders) == n_orders
        assert all(_native.gpu_lib().nrtgpu_sort_order_device_bytes(h) == 8 * N_DOCS for h in gix._orders.values())
        res = s.search_sorted(qs, SortFieldCollector(40, spec, terminate_after=100))
        assert res.terminated_early[3] == 1 and res.relation[3] == 1
        lib = _native.gpu_lib()
        carr, ncl, qarr, nq = compile_queries(qs)
        docs, vals = np.zeros((nq, 40), np.int32), np.zeros((nq, 40, 2), np.int64)
        cnt, tot, rel, to, te = (np.zeros(nq, t) for t in (np.int32, np.int64, np.uint8, np.uint8, np.uint8))
        lim = _native.SearchLimits(0.5, 1.0, 0, 0, 0)   # the request spent its budget before the call
        rc = lib.nrtgpu_search_sorted_fields(gix.handle, gix.sort_order(spec), carr, ncl, qarr, nq, 40, 0, None, C.byref(lim), None,
                                             docs.ctypes.data, vals.ctypes.data, cnt.ctypes.data, tot.ctypes.data, rel.ctypes.data,
                                             to.ctypes.data, te.ctypes.data)
        assert rc == 0 and to[3] == 1 and rel[3] == 1
    finally:
        gix.close()


def test_refusals(setup, leaves):
    sh, qs, gix = setup
    ls, s = leaves
    lib = _native.gpu_lib()
    F = _native.SortField
    INVALID = 1

    def create(fields, index=gix):
        arr = (F * len(fields))(*fields)
        h = C.c_void_p()
        rc = lib.nrtgpu_sort_order_create(index.handle, arr, len(fields), None, C.byref(h))
        msg = _native.gpu_lib().nrtgpu_last_error().decode() if rc else ""
        if rc == 0:
            lib.nrtgpu_sort_order_close(h)
        return rc, msg

    assert create([F(5, KW_SET, 0, 4, 0)]) == (INVALID, "bad sort selector")
    assert create([F(5, KW_SET, 0, -1, 0)]) == (INVALID, "bad sort selector")
    assert create([F(1, INT, 0, 2, 0)]) == (INVALID, "bad sort selector")      # MIDDLE on a numeric column
    assert create([F(5, 4, 0, 0, 0)]) == (INVALID, "keyword sort column out of range")
    assert create([F(5, KW, 0, 0, 2)])[0] == INVALID and "missing_value" in create([F(5, KW, 0, 0, 2)])[1]
    assert create([F(5, KW, 0, 3, 1)])[0] == 0   # a selector on a SORTED column is ignored
    with pytest.raises(ValueError):
        SortType(INT, field_type="int", selector="middle_min").c_field()
    # an after code beyond 2n + 1, on an image and on the leaves (reader-wide n)
    n = len(sh.keyword_columns[KW].terms)
    for searcher, hi in ((GpuIndexSearcher(gix), n), (s, n)):
        ok = searcher.search_sorted(qs[:1], SortFieldCollector(5, [K()]), search_after=[FieldDoc(0, values=(2 * hi + 1,))])
        assert ok.counts[0] == 0   # after the last term: nothing follows
        with pytest.raises(NrtGpuError, match="keyword after value"):
            searcher.search_sorted(qs[:1], SortFieldCollector(5, [K()]), search_after=[FieldDoc(0, values=(2 * hi + 2,))])
        with pytest.raises(NrtGpuError, match="keyword after value"):
            searcher.search_sorted(qs[:1], SortFieldCollector(5, [K()]), search_after=[FieldDoc(0, values=(-1,))])
    # leaves with different KEYWORD specs
    orders = (C.c_void_p * 3)(ls[0].sort_order([K()]).value, ls[1].sort_order([K(missing_last=True)]).value, ls[2].sort_order([K()]).value)
    carr, ncl, qarr, nq = compile_queries(qs[:2])
    out = [np.zeros(64, np.int64) for _ in range(7)]
    rc = lib.nrtgpu_searcher_search_sorted_fields(s.handle, orders, 3, carr, ncl, qarr, nq, 4, 0, None, None, None,
                                                  *[o.ctypes.data for o in out])
    assert rc == INVALID and "different Sorts" in lib.nrtgpu_last_error().decode()
    # the one-field path keeps refusing the KEYWORD kind
    cs = _native.Sort(5, KW, 0, 0, 0, None)
    rc = lib.nrtgpu_search_sorted(gix.handle, carr, ncl, qarr, nq, 4, 0, C.byref(cs), None, None, *[o.ctypes.data for o in out[:5]],
                                  None, None)
    assert rc == INVALID and lib.nrtgpu_last_error().decode() == "bad sort kind"
