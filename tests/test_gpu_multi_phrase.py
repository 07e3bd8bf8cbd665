"""Multi-phrase leaves on the GPU (NRTGPU_MULTI_PHRASE: union lists built by union_kernel.cuh, read by the window engine's
bool_window_union_kernel) against the CPU reference (tests/multi_phrase_reference.py), bit for bit: generated trees of
terms, phrases, multi-phrases, dismaxes and constant-score nodes at slop 0 and > 0, a 1024-query typeahead batch,
collectors, three leaves against one image, live-docs updates, repeated calls, the union cap, and multi-phrases of one
term per position against PhraseQuery."""
import os

import numpy as np
import pytest

import multi_phrase_reference as mpr
import phrase_reference as pr
import score_nodes_reference as snr
import oracle
from nrtsearch_b200 import NrtGpuError, _native
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, ConstantScoreQuery, DisjunctionMaxQuery, GpuContext, GpuIndex,
                                   GpuIndexSearcher, GpuLeafSearcher, MatchPhrasePrefixQuery, MultiPhraseQuery, Occur, PhraseQuery,
                                   RelevanceCollector, TermQuery, TermsCollector, compile_tree)

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
N_DOCS = 300_000
V0, V1 = 3000, 2000
S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
FAMILY = 60   # a "prefix" is a run of FAMILY consecutive term ids (the sorted dictionary's terms that share it)


def token_shard():
    rng = np.random.default_rng(7)
    docs, terms, poss = [], [], []
    for f, (lo, mean, vocab, base) in enumerate(((3, 5.0, V0, 0), (2, 3.0, V1, V0))):
        lens = lo + rng.poisson(mean, N_DOCS)
        start = np.zeros(N_DOCS + 1, np.int64)
        np.cumsum(lens, out=start[1:])
        w = 1.0 / np.arange(1, vocab + 1) ** 0.8
        cdf = np.cumsum(w) / w.sum()
        tok = np.searchsorted(cdf, rng.random(int(start[-1]))).astype(np.int64) + base
        doc = np.repeat(np.arange(N_DOCS), lens)
        pos = np.arange(int(start[-1])) - start[doc]
        if f == 0:   # stacked synonyms: a second token at the position of 2% of the tokens, and a few tf >= 255 docs
            st = rng.random(len(tok)) < 0.02
            hot = np.repeat(rng.choice(N_DOCS, 6, replace=False), 300)
            doc = np.concatenate([doc, doc[st], hot])
            pos = np.concatenate([pos, pos[st], np.tile(np.arange(300), 6) + 1000])
            tok = np.concatenate([tok, rng.integers(0, 200, int(st.sum())), np.full(len(hot), 1)])
        docs.append(doc), terms.append(tok), poss.append(pos)
    term_field = np.array([0] * V0 + [1] * V1, np.int32)
    sh = pr.shard_from_token_arrays(N_DOCS, term_field, 2, np.concatenate(docs), np.concatenate(terms), np.concatenate(poss),
                                    live_docs=(rng.random(N_DOCS) > 0.05).astype(np.uint8))
    sh.columns, sh.column_has = [(np.arange(N_DOCS) % 7).astype(np.int64)], [None]
    return sh


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    sh = token_shard()
    g = GpuIndex(gpu_ctx, sh)
    yield sh, g
    g.close()


def expansions(fam, n, base=0):
    return [base + fam * FAMILY + i for i in range(n)]


def prefix(tokens, fam, n=50, slop=0, base=0):
    return MatchPhrasePrefixQuery([[base + t] for t in tokens], expansions(fam, n, base), slop)


def queries(seed, n):
    rng = np.random.default_rng(seed)

    def leaf():
        f = int(rng.integers(0, 2))
        base, vocab = (0, V0) if f == 0 else (V0, V1)
        r = rng.random()
        if r < 0.2:
            return TermQuery(base + int(rng.integers(0, 300)))
        if r < 0.35:
            a, b = (base + int(t) for t in rng.integers(0, 40, 2))
            return PhraseQuery([a, b], slop=int(rng.integers(0, 3)) if a != b else 0)
        if r < 0.7:
            toks = [int(t) for t in rng.integers(0, 60, int(rng.integers(0, 3)))]
            slop = int(rng.integers(1, 3)) if rng.random() < 0.3 else 0
            fam = int(rng.integers(0, vocab // FAMILY))
            alts = expansions(fam, int(rng.integers(1, FAMILY + 1)), base)
            if slop and (set(toks) & set(alts) or len(set(toks)) < len(toks)):
                slop = 0
            return MatchPhrasePrefixQuery([[base + t] for t in toks], alts, slop)
        k = int(rng.integers(2, 4))
        arrays = [[base + int(t) for t in rng.integers(0, 200, int(rng.integers(1, 4)))] for _ in range(k)]
        slop = int(rng.integers(1, 3)) if rng.random() < 0.3 else 0
        flat = [t for a in arrays for t in a]
        if slop and len(set(flat)) < len(flat):
            slop = 0
        return MultiPhraseQuery(arrays, slop=slop)

    def node(depth, slots):   # slots: [term slots, nested nodes] used so far
        kids = []
        for _ in range(int(rng.integers(1, 4))):
            if depth < 1 and rng.random() < 0.3 and slots[1] < 4:
                slots[1] += 1
                kids.append(node(depth + 1, slots))
            else:
                q = leaf()
                need = 1 if isinstance(q, TermQuery) else len(q.terms) + (1 if isinstance(q, MatchPhrasePrefixQuery) else 0)
                if slots[0] + need > 6:   # (room for the two term leaves a node may add below)
                    continue
                slots[0] += need
                kids.append(q)
        kids = kids or [TermQuery(5)]
        r = rng.random()
        if r < 0.25:
            return DisjunctionMaxQuery(kids, float(rng.choice([0.0, 0.25])))
        if r < 0.35 and depth > 0 and slots[1] < 8:
            slots[1] += 1
            return BoostQuery(ConstantScoreQuery(kids[0]), 2.5)
        b = BooleanQuery()
        for k in kids:
            if rng.random() < 0.15 and slots[1] < 8 and not isinstance(k, (BooleanQuery, DisjunctionMaxQuery, BoostQuery)):
                slots[1] += 1
                k = ConstantScoreQuery(k)
            b.add(BoostQuery(k, float(rng.choice([1.0, 1.0, 0.5, 3.0]))), Occur(int(rng.choice([0, 0, 0, 1, 2, 3]))))
        if all(c.occur == N for c in b.clauses):
            b.add(TermQuery(7), S)
        return b

    return [node(0, [0, 0]) for _ in range(n)]


def check(res, want, k, what=""):
    for q in range(len(res.counts)):
        n = min(int(want[2][q]), k)
        assert res.counts[q] == n, f"{what} query {q}: counts {res.counts[q]} vs {n}"
        assert np.array_equal(res.docs[q, :n], want[0][q, :n]), f"{what} query {q}: docs differ"
        assert np.array_equal(res.scores[q, :n].view(np.uint32), want[1][q, :n].view(np.uint32)), f"{what} query {q}: scores differ"
    assert np.array_equal(res.total_hits, want[3]), f"{what}: totalHits differ"


@pytest.fixture(scope="module")
def trees(corpus):
    sh, _ = corpus
    qs = queries(3, 160) + [prefix([], 2), prefix([0], 1), prefix([3, 4], 2, slop=1), prefix([0], 4, n=1),
                            MultiPhraseQuery([[0, 200], [1]]), MatchPhrasePrefixQuery([[0]], []), MultiPhraseQuery([])]
    return qs, mpr.search(sh, qs, 100)


@pytest.mark.parametrize("k", [10, 100])
def test_trees_equal_the_reference(corpus, trees, k):
    sh, g = corpus
    qs, want = trees
    assert (want[3] > 0).sum() > len(qs) // 2
    check(GpuIndexSearcher(g).search_tree(qs, RelevanceCollector(k, INT_MAX)), want, k)


def test_a_repeated_call_is_identical(corpus, trees):
    _, g = corpus
    qs, _ = trees
    a = GpuIndexSearcher(g).search_tree(qs, RelevanceCollector(50, INT_MAX))
    b = GpuIndexSearcher(g).search_tree(qs, RelevanceCollector(50, INT_MAX))
    p = GpuIndexSearcher(g).prepare_tree(qs, RelevanceCollector(50, INT_MAX))
    try:
        p.run()
        c = p.fetch()
        p.run()
        d = p.fetch()
    finally:
        p.close()
    for x in (b, c, d):
        for f in ("docs", "scores", "counts", "total_hits"):
            assert np.array_equal(getattr(a, f), getattr(x, f)), f


def test_typeahead_batch(corpus):
    """1024 queries of one and two tokens, each prefix expanded to 50 terms: 8 distinct prefixes, so the batch builds
    few unions however many queries share them"""
    sh, g = corpus
    rng = np.random.default_rng(5)
    shapes = [prefix([], f) for f in range(4)] + [prefix([t], f) for t, f in ((0, 0), (1, 2), (4, 1), (2, 3))]
    qs = [shapes[int(i)] for i in rng.integers(0, len(shapes), 1024)]
    want_one = mpr.search(sh, shapes, 10)
    res = GpuIndexSearcher(g).search_tree(qs, RelevanceCollector(10, INT_MAX))
    idx = [shapes.index(q) for q in qs]
    want = tuple(w[idx] for w in want_one)
    check(res, want, 10, "typeahead")
    assert (want_one[3] > 0).all()


def test_with_collectors(corpus, trees):
    sh, g = corpus
    qs, want = trees
    qs, want = qs[:40], tuple(w[:40] for w in want)
    res, outs = GpuIndexSearcher(g).search_tree_with_collectors(qs, RelevanceCollector(10, INT_MAX), [TermsCollector(0, 7)])
    check(res, want, 10, "collectors")
    carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(qs, phrase_table=True)
    leaves = mpr.MultiPhraseLeaves(sh, oracle.OracleIndex(sh), parr, tarr)
    for q in range(nq):
        p, _ = snr.evaluate(sh, carr, narr, qarr[q].clause_begin, qarr[q].clause_end, qarr[q].min_should_match, leaves)
        counts = np.bincount(sh.columns[0][p & leaves.live], minlength=7)
        o = outs[0]
        got = {int(o["keys"][q, j]): int(o["counts"][q, j]) for j in range(int(o["n"][q]))}
        assert got == {v: int(c) for v, c in enumerate(counts) if c}, f"query {q}"


def test_three_leaves_equal_one_image(gpu_ctx, corpus, trees):
    sh, _ = corpus
    qs, want = trees
    cuts = [0, 70_001, 200_000, N_DOCS]
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    try:
        res = GpuLeafSearcher(gpu_ctx, leaves).search_tree(qs, RelevanceCollector(100, INT_MAX))
        check(res, want, 100, "leaves")
    finally:
        for g in leaves:
            g.close()


def test_live_docs_updates(gpu_ctx, corpus, trees):
    sh, _ = corpus
    qs, _ = trees
    g = GpuIndex(gpu_ctx, sh)
    try:
        p = GpuIndexSearcher(g).prepare_tree(qs, RelevanceCollector(20, INT_MAX))   # unions built before the update
        live = (np.random.default_rng(9).random(N_DOCS) > 0.3).astype(np.uint8)
        g.set_live_docs(live)
        sh2 = sh.doc_range(0, N_DOCS)
        sh2.live_docs = live
        want = mpr.search(sh2, qs, 20)
        check(GpuIndexSearcher(g).search_tree(qs, RelevanceCollector(20, INT_MAX)), want, 20, "after")
        p.run()
        check(p.fetch(), want, 20, "prepared")
        p.close()
    finally:
        g.close()


def test_one_term_per_position_is_the_phrase(corpus):
    _, g = corpus
    rng = np.random.default_rng(13)
    ps = []
    for i in range(60):
        # every other phrase repeats a term (exact only: a sloppy repeat is refused); both count its idf each time
        terms = [int(t) for t in rng.choice(50, int(rng.integers(2, 5)), replace=False)]
        if i % 2:
            terms.append(terms[0])
        ps.append((terms, 0 if i % 2 else int(rng.integers(0, 3))))
    s = GpuIndexSearcher(g)
    a = s.search_tree([MultiPhraseQuery([[t] for t in t_], slop=sl) for t_, sl in ps], RelevanceCollector(100, INT_MAX))
    b = s.search_tree([PhraseQuery(t_, slop=sl) for t_, sl in ps], RelevanceCollector(100, INT_MAX))
    for f in ("docs", "scores", "counts", "total_hits"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f


def test_the_union_cap_refuses_cleanly(corpus):
    sh, _ = corpus
    os.environ["NRTGPU_UNION_POSTINGS"] = "1000"
    try:
        ctx = GpuContext(0)
    finally:
        del os.environ["NRTGPU_UNION_POSTINGS"]
    g = GpuIndex(ctx, sh)
    try:
        s = GpuIndexSearcher(g)
        with pytest.raises(NrtGpuError) as e:
            s.search_tree([prefix([], 0)], RelevanceCollector(10, INT_MAX))
        assert e.value.status == 3 and "more than 1000" in str(e.value)
        # the raw call writes none of its outputs
        a = compile_tree([prefix([], 0), TermQuery(3)], phrase_table=True)
        nq, k = a[9], 10
        outs = [np.full(nq * k, -7, np.int32), np.full(nq * k, -7.0, np.float32), np.full(nq, -7, np.int32),
                np.full(nq, -7, np.int64), np.full(nq, 7, np.uint8), np.full(nq, 7, np.uint8), np.full(nq, 7, np.uint8)]
        rc = _native.gpu_lib().nrtgpu_search_tree_phrases(g.handle, *a[:9], nq, k, INT_MAX, 0, None, None,
                                                           *[o.ctypes.data for o in outs])
        assert rc == 3
        for o in outs:
            assert (o == o.flat[0]).all() and o.flat[0] in (-7, 7)
        res = s.search_tree([prefix([], 0, n=1), PhraseQuery([0, 1])], RelevanceCollector(10, INT_MAX))   # no union: fine
        assert res.counts.all()
    finally:
        g.close()
        ctx.close()
