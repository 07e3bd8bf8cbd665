"""Terms aggregations over keyword columns on the GPU path (nrtgpu_index_add_keyword_columns, value_type 3 on a TERMS
record, TermsCollector(field_type="keyword")) against tests/keyword_aggs_reference.py, fed with
rescore_tree_reference.evaluate_all: the match set and float32 score of every query over every doc, deletes applied.

The shard is tests/test_gpu_tree_aggs.py's (tests/test_gpu_phrase.py's 1.25M docs with positions and its numeric columns)
with 8 % deletes and two keyword columns: SORTED over 500 terms (ASCII, Latin-1 and 4-byte UTF-8, so byte order is not
code-point-by-code-unit order) with 10 % of docs without a value, and SORTED_SET of 0-4 Zipf-drawn terms of 2,000 per doc,
drawn with repeats that the column's set collapses, plus 40 docs of 9 to 60 terms; later docs draw from more terms, so the leaves' dictionaries differ. Collectors: keyword terms desc / asc at size 1, 10 and 2048 with nested
min / max / sum, top hits by score and by a Sort, buckets ordered by a nested value, and keyword terms under a query filter
and a numeric value-set filter, on the probe kernel (flat batches) and the window engine (trees, phrases, a wide flat
batch). Keys, counts, totalBuckets, otherCounts, min / max, top-hit docs, score bits and sort values are exact, sums within
aggs_reference's bound. Three doc-range leaves, each with its own dictionary, equal the whole shard; a repeated call is
identical."""
import dataclasses

import numpy as np
import pytest

import keyword_aggs_reference as kr
import oracle
import test_gpu_tree_aggs as ta
from nrtsearch_b200 import NrtGpuError, _native
from nrtsearch_b200._native import check as check_rc
from nrtsearch_b200.index import KeywordColumn, PinnedDesc
from nrtsearch_b200.search import (FilterCollector, GpuIndex, GpuIndexSearcher, GpuLeafSearcher, MaxCollector, MinCollector,
                                   RangeQuery, RelevanceCollector, SortType, SumCollector, TermsCollector, TopHitsCollector,
                                   ValueSetFilter)
from test_gpu_phrase import token_shard

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
KW_ONE, KW_SET = 0, 1      # keyword columns
CAT, DBL = ta.CAT, ta.DBL  # numeric columns of add_columns
CUTS = [0, 300_017, 870_000]


def keyword_columns(n):
    rng = np.random.default_rng(0x4B57)
    alphabet = ["pizza", "sushi", "tacos", "café", "Zürich", "naïve", "\U0001f355", "b", "B", "ab", "a"]
    words = sorted({f"{alphabet[i % len(alphabet)]}-{i:04d}" for i in range(500)})
    # later docs draw from more terms, so each doc-range leaf has a dictionary of its own
    one_lim = 200 + (np.arange(n) * 300) // n
    one = [None if rng.random() < 0.1 else words[int(rng.integers(0, one_lim[d]))] for d in range(n)]
    pool = [f"cat/{i:05d}" + ("é" if i % 7 == 0 else "") for i in range(2000)]
    z = rng.zipf(1.3, size=4 * n)
    set_lim = 600 + (np.arange(n) * 1400) // n
    per = rng.integers(0, 5, n)
    start = np.concatenate([[0], np.cumsum(per)[:-1]])
    sets = [[pool[int(z[s + k] % set_lim[d])] for k in range(p)] + ([pool[int(z[s] % set_lim[d])]] if p and d % 5 == 0 else [])
            for d, (s, p) in enumerate(zip(start, per))]   # (the repeats collapse in the column's set)
    for d in range(7, n, n // 40):   # a few docs of many terms: 9 to 60 each
        sets[d] = pool[(d % 300): (d % 300) + 9 + d % 52]
    return [KeywordColumn.from_values(one, False), KeywordColumn.from_values(sets, True)]


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    sh = ta.add_columns(token_shard())
    sh.live_docs = (np.random.default_rng(0x8D).random(sh.n_docs) >= 0.08).astype(np.uint8)
    sh.keyword_columns = keyword_columns(sh.n_docs)
    assert max(np.diff(sh.keyword_columns[KW_SET].offsets)) > 8
    g = GpuIndex(gpu_ctx, sh)
    yield sh, oracle.OracleIndex(sh), g
    g.close()


@pytest.fixture(scope="module")
def leaves(gpu_ctx, corpus):
    sh = corpus[0]
    cuts = CUTS + [sh.n_docs]
    ls = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    s = GpuLeafSearcher(gpu_ctx, ls)
    yield ls, s
    s.close()
    for g in ls:
        g.close()


SORT = SortType(CAT, field_type="int", reverse=True)
FILTER_Q = RangeQuery(0, 200_000, 900_000)
FILTER_SET = ValueSetFilter(CAT, (3, 4, 5, 17, -2), "int")


def collector_groups():
    """three requests, together covering every collector shape"""
    return [
        [TermsCollector(KW_ONE, 10, field_type="keyword", nested=(("mx", MaxCollector(DBL, "double")), ("s", SumCollector(0)),
                                                                   ("top", TopHitsCollector(3)))),
         TermsCollector(KW_SET, 2048, order_desc=False, field_type="keyword",
                        nested=(("mn", MinCollector(CAT, "int")), ("srt", TopHitsCollector(4, 1, SORT)), ("top", TopHitsCollector(2)))),
         FilterCollector(FILTER_SET, (("t", TermsCollector(KW_ONE, 5, field_type="keyword", nested=(("top", TopHitsCollector(2)),))),))],
        [TermsCollector(KW_SET, 1, field_type="keyword", nested=(("mx", MaxCollector(DBL, "double")), ("top", TopHitsCollector(3))),
                        order_by="mx"),
         TermsCollector(KW_ONE, 2048, order_desc=False, field_type="keyword", nested=(("mn", MinCollector(0)),), order_by="mn")],
        [FilterCollector(FILTER_Q, (("t", TermsCollector(KW_SET, 7, field_type="keyword", nested=(("s", SumCollector(0)),
                                                                                                    ("top", TopHitsCollector(3))))),
                                    ("n", TermsCollector(CAT, 4, field_type="int"))))],
    ]


def check(R, q, c, o, sel, what):
    """ta.check, with keyword terms collectors checked against keyword_aggs_reference"""
    if isinstance(c, FilterCollector):
        b = sel & R.mask(c.filter)
        assert o["doc_count"][q] == b.sum(), f"{what}: doc_count"
        for name, x in c.nested:
            check(R, q, x, o[name], b, f"{what}/{name}")
        return
    if not (isinstance(c, TermsCollector) and c.field_type == "keyword"):
        return ta.check(R, q, c, o, sel, what)
    specs = {name: ("min" if isinstance(x, MinCollector) else "max" if isinstance(x, MaxCollector) else "sum", x.column,
                    ta.VT[x.field_type]) for name, x in c.nested if not isinstance(x, TopHitsCollector)}
    want = kr.terms_nested(R.sh, R.sh.keyword_columns[c.column], sel, c.size, c.order_desc, specs, c.order_by, R.score[q])
    n = want["n"]
    assert o["n"][q] == n and o["total_buckets"][q] == want["total_buckets"], f"{what}: buckets"
    assert o["keys"][q][:n].tolist() == want["keys"] and all(k is None for k in o["keys"][q][n:]), f"{what}: keys"
    assert o["counts"][q][:n].tolist() == want["counts"].tolist(), f"{what}: counts"
    assert o["other_counts"][q] == want["other_counts"], f"{what}: other_counts"
    for name, x in c.nested:
        for i in range(n):
            if isinstance(x, TopHitsCollector):
                b = np.zeros(R.sh.n_docs, bool)
                b[want["members"][i]] = True
                ta.check_hits(o["nested"][name], (q, i), R, q, x, b, f"{what}/{name} slot {i}")
            else:
                ta.value_ok(float(o["nested"][name][q, i]), want["nested"][name][i], f"{what}/{name} slot {i}")


def same_outs(a, b, what):
    """two collector results equal element by element (keyword keys as str, floats by their bits)"""
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for key in a:
            same_outs(a[key], b[key], f"{what}/{key}")
    elif np.asarray(a).dtype == object:
        assert np.asarray(a).tolist() == np.asarray(b).tolist(), what
    else:
        assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)), what


def check_all(R, res, outs, colls, what):
    for q in range(len(res.counts)):
        for c, o in zip(colls, outs):
            check(R, q, c, o, R.present[q], f"{what} query {q} {type(c).__name__}")
        assert res.total_hits[q] == R.present[q].sum(), f"{what} query {q}: totalHits"


BATCHES = {"flat": ta.NARROW, "trees": ta.TREES, "wide": ta.SIX}


@pytest.fixture(scope="module")
def refs(corpus):
    sh, oix, _ = corpus
    return {name: ta.Ref(sh, oix, qs) for name, qs in BATCHES.items()}


def run(searcher, name, colls, tree):
    fn = searcher.search_tree_with_collectors if tree else searcher.search_with_collectors
    return fn(BATCHES[name], RelevanceCollector(10, INT_MAX), colls)


@pytest.mark.parametrize("name,tree", [("flat", False), ("flat", True), ("trees", True), ("wide", True)])
def test_one_image_against_the_reference(corpus, refs, name, tree):
    g = GpuIndexSearcher(corpus[2])
    for colls in collector_groups():
        res, outs = run(g, name, colls, tree)
        check_all(refs[name], res, outs, colls, f"{name} tree={tree}")


@pytest.mark.parametrize("name,tree", [("flat", False), ("trees", True)])
def test_three_leaves_equal_the_whole_image(corpus, leaves, refs, name, tree):
    ls, s = leaves
    parts = [corpus[0].doc_range(a, b) for a, b in zip(CUTS, CUTS[1:] + [corpus[0].n_docs])]
    for k in (KW_ONE, KW_SET):   # every leaf numbers its own dictionary; none is the union
        sizes = [len(p.keyword_columns[k].terms) for p in parts]
        assert len(set(sizes)) == 3 and max(sizes[:2]) < len(corpus[0].keyword_columns[k].terms), sizes
    whole = GpuIndexSearcher(corpus[2])
    for colls in collector_groups():
        res, outs = run(s, name, colls, tree)
        check_all(refs[name], res, outs, colls, f"leaves {name}")
        wres, wouts = run(whole, name, colls, tree)
        ta.same_page(res, wres, f"leaves {name}")


def test_repeat_is_identical(corpus, leaves):
    for searcher in (GpuIndexSearcher(corpus[2]), leaves[1]):
        for colls in collector_groups():
            a = run(searcher, "trees", colls, True)
            b = run(searcher, "trees", colls, True)
            ta.same_page(a[0], b[0], "repeat")
            for x, y in zip(a[1], b[1]):
                same_outs(x, y, "repeat")


def test_term_accessors_and_device_bytes(gpu_ctx, corpus, leaves):
    sh, _, g = corpus
    for k, col in enumerate(sh.keyword_columns):
        for o in (0, len(col.terms) // 2, len(col.terms) - 1):
            assert g.keyword_term(k, o) == col.terms[o]
    uni = kr.union([l.keyword_columns[KW_SET] for l in [sh.doc_range(a, b) for a, b in zip(CUTS, CUTS[1:] + [sh.n_docs])]])
    assert uni == sh.keyword_columns[KW_SET].terms
    assert [leaves[1].keyword_term(KW_SET, o) for o in (0, 7, len(uni) - 1)] == [uni[0], uni[7], uni[-1]]
    small = sh.doc_range(0, 1000)
    plain = GpuIndex(gpu_ctx, dataclasses.replace(small, keyword_columns=[]))
    with_kw = GpuIndex(gpu_ctx, small)
    # SORTED: 4 B per doc; SORTED_SET: 4 B per value and the int64 doc offsets
    n_values = int(small.keyword_columns[KW_SET].offsets[-1])
    assert with_kw.device_bytes - plain.device_bytes == 4 * 1000 + 4 * n_values + 8 * 1001
    p = PinnedDesc(small)   # an image takes its keyword columns once
    with pytest.raises(NrtGpuError, match="already has its keyword columns"):
        check_rc(_native.gpu_lib().nrtgpu_index_add_keyword_columns(with_kw.handle, p.keyword, p.n_keyword))
    with pytest.raises(NrtGpuError, match="bad aggregation value_type"):
        GpuIndexSearcher(with_kw).search_with_collectors(ta.NARROW, RelevanceCollector(10, INT_MAX), [MaxCollector(KW_ONE, "keyword")])
    plain.close()
    with_kw.close()
