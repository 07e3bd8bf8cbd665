"""Keyword range and prefix queries (NRTGPU_KEYWORD_RANGE clauses) and keyword value sets (NRTGPU_AGG_FILTER_KEYWORD_SET) on
the GPU path.

Parity through shadow columns: the shard's keyword columns (SORTED, thousands of terms, ~5 % of docs without a value;
SORTED_SET, 0-5 terms per doc) are mirrored as numeric columns of their codes (single-valued with has = code != 0, and
multi-valued). A batch whose keyword clauses are replaced by NRTGPU_RANGE_I64 clauses on the shadow column over the same
codes must give bit-identical docs, score bits, counts, totalHits, relation and flags, on every entry point, and the shadow
batch matches the oracle. The code ranges themselves are tied to bytes by tests/keyword_query_reference.py. Searchers over
leaves whose dictionaries differ must equal one image of the whole shard."""
import ctypes as C

import numpy as np
import pytest

import keyword_query_reference as kr
import oracle
from nrtsearch_b200 import NrtGpuError, _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200.index import KeywordColumn
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, FilterCollector, GpuBatcher, GpuIndex,
                                   GpuIndexSearcher, GpuLeafSearcher, KeywordPrefixQuery, KeywordRangeQuery, MatchAllDocsQuery,
                                   Occur, PhraseQuery, RangeQuery, RelevanceCollector, ScoreDoc, SortFieldCollector, SortType,
                                   TermQuery, TermsCollector, TopHitsCollector, ValueSetFilter, _KeywordCodes, compile_queries)

pytestmark = pytest.mark.gpu

N_DOCS, VOCAB, DIMS = 300_000, 6_000, 32
KW, KW_SET = 0, 1                       # keyword columns
SHADOW = {KW: 0, KW_SET: 1}             # their numeric shadows
INT = 2                                 # a numeric column 0..99
INT_MAX = 2**31 - 1
OCC = [Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT]


def words():
    w = {"", "a", "a\x00", "ab", "\xff", "zz", "prefix1a", "prefix1b", "prefix2a"}
    for i in range(4000):
        w.add(f"{'abcdefgh'[i % 8]}{'xyz'[i % 3]}{i:04d}")
    return sorted(w, key=lambda s: s.encode())


WORDS = words()


def make_shard():
    sh = ix.synth_text_shard(N_DOCS, VOCAB, min_len=6, poisson_mean=20.0)
    rng = np.random.default_rng(0xC0DE)
    # the SORTED column draws from the first 60 % of the words for the first half of the docs (so the leaves' dictionaries differ)
    lim = np.where(np.arange(N_DOCS) < N_DOCS // 2, int(len(WORDS) * 0.6), len(WORDS))
    one = [None if rng.random() < 0.05 else WORDS[int(rng.integers(0, lim[d]))] for d in range(N_DOCS)]
    per = rng.integers(0, 6, N_DOCS)
    sets = [[WORDS[int(x)] for x in rng.integers(len(WORDS) // 3, len(WORDS), p)] if d >= 200_000 else
            [WORDS[int(x)] for x in rng.integers(0, len(WORDS), p)] for d, p in enumerate(per)]
    kc = [KeywordColumn.from_values(one, False), KeywordColumn.from_values(sets, True)]
    codes_one = np.where(kc[0].ords < 0, 0, 2 * kc[0].ords.astype(np.int64) + 2)
    sh.columns = [codes_one, 2 * kc[1].ords.astype(np.int64) + 2, rng.integers(0, 100, N_DOCS).astype(np.int64)]
    sh.column_has = [(codes_one != 0).astype(np.uint8), None, None]
    sh.column_offsets = [None, kc[1].offsets, None]
    sh.keyword_columns = kc
    sh.live_docs = (rng.random(N_DOCS) < 0.93).astype(np.uint8)
    sh.vectors = ix.synth_vectors(N_DOCS, DIMS)
    sh.vec_similarity = ix.SIM_COSINE
    f = sh.post_freqs.astype(np.int64)   # positions: posting p holds freq ascending positions
    start = np.repeat(np.cumsum(f) - f, f)
    sh.post_positions = (2 * (np.arange(int(f.sum())) - start) + np.repeat(sh.post_docs % 3, f)).astype(np.int32)
    return sh


@pytest.fixture(scope="module")
def shard():
    return make_shard()


@pytest.fixture(scope="module")
def image(gpu_ctx, shard):
    g = GpuIndex(gpu_ctx, shard)
    yield g
    g.close()


@pytest.fixture(scope="module")
def oix(shard):
    return oracle.OracleIndex(shard)


def twin(q, image):
    """q with every keyword query replaced by the RangeQuery on its shadow column over the image's code range"""
    if isinstance(q, (KeywordRangeQuery, KeywordPrefixQuery)):
        lo, hi = image.keyword_range(q)
        return RangeQuery(SHADOW[q.column], lo, hi)
    if isinstance(q, _KeywordCodes):
        return RangeQuery(SHADOW[q.column], q.lo, q.hi)
    if isinstance(q, BoostQuery):
        return BoostQuery(twin(q.query, image), q.boost)
    if isinstance(q, BooleanQuery):
        b = BooleanQuery(minimum_number_should_match=q.minimum_number_should_match)
        for c in q.clauses:
            b.add(twin(c.query, image), c.occur)
        return b
    if isinstance(q, DisjunctionMaxQuery):
        return DisjunctionMaxQuery([twin(d, image) for d in q.disjuncts], q.tie_breaker)
    if isinstance(q, FilterCollector):
        f = q.filter
        if isinstance(f, ValueSetFilter) and f.field_type == "keyword":
            f = ValueSetFilter(SHADOW[f.column], tuple(image.keyword_seek(f.column, v.encode()) for v in f.values))
        else:
            f = twin(f, image)
        return FilterCollector(f, tuple((n, twin(c, image)) for n, c in q.nested))
    return q


def rand_kw(rng):
    """a keyword range or prefix query on one of the two columns, with bounds held, missing or outside every term"""
    col = int(rng.integers(0, 2))
    r = rng.random()
    pick = lambda: WORDS[int(rng.integers(0, len(WORDS)))] + ("" if rng.random() < 0.7 else "m")
    if r < 0.25:
        return KeywordPrefixQuery(col, pick()[:int(rng.integers(0, 3))])
    lo, hi = sorted([pick(), pick()], key=lambda s: s.encode())
    if rng.random() < 0.1:
        lo, hi = hi, lo   # lower > upper: matches nothing
    return KeywordRangeQuery(col, None if rng.random() < 0.15 else lo, None if rng.random() < 0.15 else hi,
                             bool(rng.random() < 0.6), bool(rng.random() < 0.6))


def make_queries(n, seed, n_terms=(1, 3), keyword_only=False):
    rng = np.random.default_rng(seed)
    terms = ix.synth_query_terms(n, 8, VOCAB, seed=seed, log10_lo=0.5, log10_hi=3.5)
    qs = []
    for i in range(n):
        b = BooleanQuery()
        nt = 0 if keyword_only else int(rng.integers(n_terms[0], n_terms[1] + 1))
        for t in terms[i][:nt]:
            b.add(TermQuery(int(t)), OCC[int(rng.integers(0, 2))] if rng.random() < 0.8 else Occur.SHOULD)
        for _ in range(int(rng.integers(1, 3))):
            k = rand_kw(rng)
            if rng.random() < 0.3:
                k = BoostQuery(k, float(rng.choice([0.5, 2.0, 3.25])))
            b.add(k, OCC[int(rng.integers(0, 4))])
        if all(c.occur == Occur.MUST_NOT for c in b.clauses):
            b.add(MatchAllDocsQuery(), Occur.FILTER)
        n_should = sum(c.occur == Occur.SHOULD for c in b.clauses)
        if n_should >= 2 and rng.random() < 0.25:
            b.minimum_number_should_match = 2
        qs.append(b)
    return qs


def deep_eq(a, b) -> bool:
    """collector results equal: dicts and lists member by member, arrays by value (floats by their bits)"""
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(deep_eq(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(deep_eq(x, y) for x, y in zip(a, b))
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind == "f":
        return a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))
    return a.shape == b.shape and bool((a == b).all())


def same(a, b, what=""):
    for name in ("docs", "counts", "total_hits", "relation", "hit_timeout", "terminated_early"):
        x, y = getattr(a, name, None), getattr(b, name, None)
        if x is not None:
            assert np.array_equal(x, y), f"{what}: {name} differ"
    assert np.array_equal(a.scores.view(np.uint32), b.scores.view(np.uint32)), f"{what}: scores differ"


def test_code_ranges_match_the_bytes_reference(image, shard, oix):
    """a keyword query's shadow range matches exactly the docs the bytes reference does (deletes aside)"""
    rng = np.random.default_rng(5)
    qs = [rand_kw(rng) for _ in range(40)] + [KeywordPrefixQuery(KW, "prefix1"), KeywordPrefixQuery(KW_SET, ""),
                                              KeywordRangeQuery(KW, "\xff", None), KeywordRangeQuery(KW_SET, None, "")]
    carr, _, qarr, _ = compile_queries([twin(q, image) for q in qs])
    live = shard.live_docs.astype(bool)
    for i, q in enumerate(qs):
        col = shard.keyword_columns[q.column]
        enc = lambda v: None if v is None else v.encode()
        pred = kr.prefix_pred(q.prefix.encode()) if isinstance(q, KeywordPrefixQuery) else \
            kr.range_pred(enc(q.lower), enc(q.upper), q.include_lower, q.include_upper)
        want = kr.match_mask(col, pred) & live
        assert np.array_equal(oracle.match_bitmap(oix, carr, qarr, i).astype(bool), want), q


@pytest.mark.parametrize("threshold", [1000, INT_MAX])
def test_flat_batches(image, oix, threshold):
    s = GpuIndexSearcher(image)
    qs = make_queries(256, 11) + make_queries(64, 12, keyword_only=True)
    coll = RelevanceCollector(20, threshold)
    a = s.search_batch(qs, coll)
    tw = [twin(q, image) for q in qs]
    b = s.search_batch(tw, coll)
    same(a, b, "flat")
    if threshold == INT_MAX:
        carr, ncl, qarr, nq = compile_queries(tw)
        wd, ws, wc, wt, wr = oracle.search_compiled(oix, carr, ncl, qarr, nq, 20)
        assert np.array_equal(b.counts, wc) and np.array_equal(b.docs, wd) and np.array_equal(b.total_hits, wt)
        assert np.array_equal(b.scores.view(np.uint32), ws.view(np.uint32))
    # searchAfter: the page after each query's 10th hit
    after = [ScoreDoc(int(a.docs[q, 9]), float(a.scores[q, 9])) if a.counts[q] >= 10 else None for q in range(len(qs))]
    same(s.search_batch(qs, coll, search_after=after), s.search_batch(tw, coll, search_after=after), "after")
    pb = s.prepare(qs, coll)
    pb.run()
    same(pb.fetch(), b, "prepared")
    pb.close()


def test_wide_batches(image):
    s = GpuIndexSearcher(image)
    qs = make_queries(64, 21, n_terms=(5, 7))
    for k in (513, 1024):
        coll = RelevanceCollector(k, INT_MAX)
        same(s.search_batch(qs, coll), s.search_batch([twin(q, image) for q in qs], coll), f"wide {k}")


def test_sorted_search_with_a_keyword_sort(image):
    s = GpuIndexSearcher(image)
    qs = make_queries(64, 31)
    coll = SortFieldCollector(30, [SortType(INT), SortType(KW, True, False, "keyword")])
    a, b = s.search_sorted(qs, coll), s.search_sorted([twin(q, image) for q in qs], coll)
    assert np.array_equal(a.docs, b.docs) and np.array_equal(a.counts, b.counts) and np.array_equal(a.total_hits, b.total_hits)
    assert (a.sort_values == b.sort_values).all()


def test_trees_with_phrases(image):
    s = GpuIndexSearcher(image)
    rng = np.random.default_rng(41)
    terms = ix.synth_query_terms(48, 4, VOCAB, seed=41, log10_lo=1.0, log10_hi=3.5)
    qs = []
    for t in terms:
        a, b, c, d = (int(x) for x in t)
        inner = DisjunctionMaxQuery([TermQuery(a), BoostQuery(rand_kw(rng), 1.5), PhraseQuery([b, c], slop=int(rng.integers(0, 3)))], 0.3)
        qs.append(BooleanQuery().add(inner, Occur.MUST).add(rand_kw(rng), OCC[int(rng.integers(0, 4))])
                  .add(BooleanQuery().add(TermQuery(d), Occur.SHOULD).add(rand_kw(rng), Occur.SHOULD), Occur.SHOULD))
    coll = RelevanceCollector(15, INT_MAX)
    same(s.search_tree(qs, coll), s.search_tree([twin(q, image) for q in qs], coll), "tree")


def test_collectors(image):
    s = GpuIndexSearcher(image)
    qs = make_queries(32, 51)
    nested = (("by_kw", TermsCollector(KW, 8, field_type="keyword", nested=(("top", TopHitsCollector(3)),))),)
    add = [FilterCollector(BooleanQuery().add(KeywordPrefixQuery(KW_SET, "a"), Occur.SHOULD)
                           .add(KeywordRangeQuery(KW, "c", "e"), Occur.SHOULD), nested),
           FilterCollector(ValueSetFilter(KW_SET, tuple(WORDS[::37]) + ("missing",), "keyword"), nested),
           FilterCollector(ValueSetFilter(KW, tuple(WORDS[5::11]), "keyword"), (("n", TermsCollector(INT, 5)),))]
    coll = RelevanceCollector(10, INT_MAX)
    a_out, a = s.search_with_collectors(qs, coll, add)
    b_out, b = s.search_with_collectors([twin(q, image) for q in qs], coll, [twin(c, image) for c in add])
    same(a_out, b_out, "collectors")
    assert deep_eq(a, b)
    assert all(int(r["doc_count"].sum()) > 0 for r in a)
    ta, tb = (s.search_tree_with_collectors(x, coll, y) for x, y in ((qs, add), ([twin(q, image) for q in qs], [twin(c, image) for c in add])))
    same(ta[0], tb[0], "window collectors")
    assert deep_eq(ta[1], tb[1])


def test_knn_filter_queries_both_paths(image, gpu_ctx):
    s = GpuIndexSearcher(image)
    nq = 24
    q = ix.synth_vectors(nq, DIMS, seed=ix.SEED_VQUERIES)
    # selective filters (the gather path) and broad ones (the candidate GEMM)
    sel = [KeywordRangeQuery(KW, WORDS[100], WORDS[101]), BooleanQuery().add(KeywordPrefixQuery(KW_SET, "ax00"), Occur.MUST)]
    broad = [KeywordRangeQuery(KW_SET, "c", None), BooleanQuery().add(KeywordPrefixQuery(KW, "a"), Occur.MUST_NOT)
             .add(MatchAllDocsQuery(), Occur.FILTER)]
    filters = [(sel + broad)[i % 4] for i in range(nq)]
    a = s.knn(q, 50, filter_queries=filters)
    g = C.c_int32()
    _native.gpu_lib().nrtgpu_knn_filter_stats(image.handle, C.byref(g), None)
    assert 0 < g.value < nq
    b = s.knn(q, 50, filter_queries=[twin(f, image) for f in filters])
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32))


def test_second_pass(image):
    s = GpuIndexSearcher(image)
    qs = make_queries(32, 61)
    first = s.search_batch(make_queries(32, 62), RelevanceCollector(100, INT_MAX))
    tw = [twin(q, image) for q in qs]
    for x, y in zip(s.score_docs(qs, first.docs, first.counts), s.score_docs(tw, first.docs, first.counts)):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
    ra = s.rescore_query(qs, first.docs, first.scores, first.counts, 50, 1.0, 2.0)
    rb = s.rescore_query(tw, first.docs, first.scores, first.counts, 50, 1.0, 2.0)
    for x, y in zip(ra, rb):
        assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32))


def test_micro_batcher(image):
    s = GpuIndexSearcher(image)
    qs = make_queries(8, 71)
    b = GpuBatcher(image, max_batch=4)
    try:
        coll = RelevanceCollector(10, 1000)
        want = s.search_batch([twin(q, image) for q in qs], coll)
        for i, q in enumerate(qs):
            td, _ = b.submit(q, coll)
            assert [d.doc for d in td.score_docs] == want.docs[i, :want.counts[i]].tolist()
            assert [np.float32(d.score) for d in td.score_docs] == want.scores[i, :want.counts[i]].tolist()
            assert td.total_hits.value == want.total_hits[i]
    finally:
        b.close()


def leaf_searcher(gpu_ctx, shard, cuts):
    leaves = [GpuIndex(gpu_ctx, shard.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    return leaves, GpuLeafSearcher(gpu_ctx, leaves)


@pytest.mark.parametrize("cuts", [[0, 150_000, N_DOCS], [0, 1, 100_000, 150_000, 200_001, N_DOCS]])
def test_searchers_equal_one_image(image, gpu_ctx, shard, cuts):
    leaves, ls = leaf_searcher(gpu_ctx, shard, cuts)
    try:
        s = GpuIndexSearcher(image)
        # bounds on terms only the second half holds, prefixes living in one leaf, and random ones
        qs = make_queries(96, 81) + [KeywordRangeQuery(KW, WORDS[int(len(WORDS) * 0.7)], WORDS[int(len(WORDS) * 0.8)], False, True),
                                     KeywordPrefixQuery(KW, WORDS[-3][:3]), KeywordPrefixQuery(KW_SET, WORDS[10][:2]),
                                     BooleanQuery().add(KeywordRangeQuery(KW, None, WORDS[-1], True, False), Occur.FILTER)]
        for thr in (1000, INT_MAX):
            coll = RelevanceCollector(25, thr)
            same(ls.search_batch(qs, coll), s.search_batch(qs, coll), f"leaves {thr}")
        coll = SortFieldCollector(20, [SortType(KW_SET, False, True, "keyword"), SortType(INT)])
        a, b = ls.search_sorted(qs, coll), s.search_sorted(qs, coll)
        assert np.array_equal(a.docs, b.docs) and (a.sort_values == b.sort_values).all() and np.array_equal(a.total_hits, b.total_hits)
        trees = [BooleanQuery().add(DisjunctionMaxQuery([q, KeywordPrefixQuery(KW, "b")], 0.5), Occur.MUST) for q in qs[:32]]
        same(ls.search_tree(trees, RelevanceCollector(10, INT_MAX)), s.search_tree(trees, RelevanceCollector(10, INT_MAX)), "tree")
        add = [FilterCollector(KeywordRangeQuery(KW, WORDS[2000], None), (("t", TermsCollector(KW_SET, 6, field_type="keyword")),)),
               FilterCollector(ValueSetFilter(KW, tuple(WORDS[-200::7]) + (WORDS[3],), "keyword"), (("m", TermsCollector(INT, 4)),))]
        coll = RelevanceCollector(10, INT_MAX)
        (ha, ra), (hb, rb) = ls.search_with_collectors(qs[:32], coll, add), s.search_with_collectors(qs[:32], coll, add)
        assert np.array_equal(ha.docs, hb.docs) and np.array_equal(ha.total_hits, hb.total_hits)
        assert deep_eq(ra, rb)
        vq = ix.synth_vectors(8, DIMS, seed=ix.SEED_VQUERIES)
        flt = [qs[i] if i % 2 else KeywordRangeQuery(KW, WORDS[2500], WORDS[2510]) for i in range(8)]
        for x, y in zip(ls.knn(vq, 20, filter_queries=flt), s.knn(vq, 20, filter_queries=flt)):
            assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32))
    finally:
        ls.close()
        for l in leaves:
            l.close()


def test_known_answers(gpu_ctx):
    """AtomFieldTest.rangeQuery and PrefixQueryTest.testAtomPrefixQuery on one image, on 6 one-doc leaves and on 2 leaves"""
    from helpers import shard_from_token_docs
    vals = list("abcdef")
    sh, _ = shard_from_token_docs([[["x"]] * 6], columns=[np.zeros(6, np.int64)])
    sh.keyword_columns = [KeywordColumn.from_values(vals, False), KeywordColumn.from_values([[v] for v in vals], True)]
    cases = [(("b", "e", True, True), "bcde"), (("b", "e", False, True), "cde"), (("b", "e", True, False), "bcd"),
             (("b", "e", False, False), "cd"), ((None, "d", True, True), "abcd"), ((None, "d", True, False), "abc"),
             (("b", None, True, True), "bcdef"), (("b", None, False, True), "cdef")]
    g = GpuIndex(gpu_ctx, sh)
    singles = [GpuIndex(gpu_ctx, sh.doc_range(i, i + 1)) for i in range(6)]
    halves = [GpuIndex(gpu_ctx, sh.doc_range(0, 2)), GpuIndex(gpu_ctx, sh.doc_range(2, 6))]
    searchers = [GpuIndexSearcher(g), GpuLeafSearcher(gpu_ctx, singles), GpuLeafSearcher(gpu_ctx, halves)]
    try:
        for s in searchers:
            for col in (0, 1):
                qs = [KeywordRangeQuery(col, lo, hi, il, iu) for (lo, hi, il, iu), _ in cases]
                r = s.search_batch(qs, RelevanceCollector(10, INT_MAX))
                for i, (_, want) in enumerate(cases):
                    assert "".join(vals[d] for d in sorted(r.docs[i, :r.counts[i]])) == want
        pv = ["prefix1a", "prefix1b", "prefix1c", "prefix2a", "prefix2b", "prefix2c", "prefix2d", "not_prefix1", "not_prefix2"]
        ps, _ = shard_from_token_docs([[["x"]] * 9], columns=[np.zeros(9, np.int64)])
        ps.keyword_columns = [KeywordColumn.from_values(pv, False)]
        pg = GpuIndex(gpu_ctx, ps)
        try:
            r = GpuIndexSearcher(pg).search_batch([KeywordPrefixQuery(0, p) for p in ("prefix1", "prefix2", "prefix", "other")],
                                                  RelevanceCollector(10, INT_MAX))
            assert [sorted(r.docs[i, :r.counts[i]].tolist()) for i in range(4)] == [[0, 1, 2], [3, 4, 5, 6], list(range(7)), []]
        finally:
            pg.close()
    finally:
        for s in searchers[1:]:
            s.close()
        for x in [g] + singles + halves:
            x.close()


def test_refusals_write_no_output(image, gpu_ctx, shard):
    L = _native.gpu_lib()
    n = len(shard.keyword_columns[KW].terms)
    for col, lo, hi, msg in ((2, 1, 1, "keyword column out of range"), (KW, 0, 5, "keyword code out of range"),
                             (KW, 1, 2 * n + 2, "keyword code out of range")):
        carr, ncl, qarr, nq = compile_queries([_KeywordCodes(col, lo, hi)])
        docs, scores, counts = np.full(5, 77, np.int32), np.full(5, 7.0, np.float32), np.full(1, 77, np.int32)
        rc = L.nrtgpu_search_bool(image.handle, carr, ncl, qarr, nq, 5, INT_MAX, 0, None, docs.ctypes.data, scores.ctypes.data,
                                  counts.ctypes.data, None, None)
        assert rc == 1 and msg in L.nrtgpu_last_error().decode()
        assert (docs == 77).all() and (scores == 7.0).all() and (counts == 77).all()
    leaves, ls = leaf_searcher(gpu_ctx, shard, [0, 150_000, N_DOCS])
    try:
        with pytest.raises(NrtGpuError, match="keyword code out of range"):
            ls.search_batch([_KeywordCodes(KW, 1, 2 * len(WORDS) + 10)], RelevanceCollector(5, INT_MAX))
        with pytest.raises(NrtGpuError, match="keyword column out of range"):
            ls.search_batch([_KeywordCodes(5, 1, 1)], RelevanceCollector(5, INT_MAX))
    finally:
        ls.close()
        for l in leaves:
            l.close()
