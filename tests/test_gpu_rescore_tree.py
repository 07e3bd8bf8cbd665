"""The second pass of tree and phrase rescore queries on the GPU (nrtgpu_score_docs_tree / nrtgpu_rescore_query_tree,
score_docs_tree_kernel) against tests/rescore_tree_reference.py, bit for bit: matches and float scores of every hit, and
the rescored pages against oracle.rescore_combine applied to that reference.

The shard: 400,000 docs at doc_base 3,000,000 built from token sequences, two text fields with positions (field 1
omitNorms), 5% deletes, an int column and a multi-valued column. Reserved field-0 terms carry planted phrases, each in a
value of its own behind the position increment gap: A (2 terms) in exactly 4096 docs, so its lists have a granule row of
the index-time skip data, B (3 terms) in exactly 4095, so its lists do not (half of them with a token between its terms),
C8 (8 terms) in 1500. The planted docs include doc 0, n_docs - 1 and docs at multiples of 1024 and one below (the first and
the last posting of their granule in A's lists). A's terms reach tf 255 and 300 in some docs, and a term is stacked at
the position of A's first term in 500 of them. Common terms have dense planes and granule rows; rare ones are short lists."""
import numpy as np
import pytest

import oracle
import phrase_reference as pr
import rescore_tree_reference as rr
from nrtsearch_b200 import NrtGpuError, NrtGpuUnsupported, _native
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, GpuIndex, GpuIndexSearcher, MatchAllDocsQuery,
                                   Occur, PhraseQuery, RangeQuery, RelevanceCollector, TermQuery, compile_tree)
from test_phrase_plan import INVALID_PHRASES, _arrays

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
N_DOCS = 400_000
DOC_BASE = 3_000_000
V0, V1 = 3000, 2000
S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
R = [V0 - 16 + i for i in range(16)]            # reserved field-0 terms: planted only
A, B, C8 = R[0:2], R[2:5], R[5:13]
STACK = R[13]                                   # stacked at the position of A's first term in 500 docs
EDGES = sorted({d for k in (0, 1, 2, 64, 200, 390) for d in (1024 * k - 1, 1024 * k) if 0 <= d < N_DOCS} | {N_DOCS - 1})
HOT = [N_DOCS - 1, 1023]                        # tf 300 of A's terms (plus others at random), docs at a granule edge
PRICE = RangeQuery(0, 100_000, 800_000)
MV = RangeQuery(1, 200, 400)                    # multi-valued column: any value
C1 = [V0 + 3, V0 + 5]                           # a common field-1 bigram (omitNorms)


def token_shard():
    rng = np.random.default_rng(43)
    docs, terms, poss = [], [], []
    for f, (lo, mean, vocab, base) in enumerate(((4, 6.0, V0, 0), (2, 4.0, V1, V0))):
        lens = lo + rng.poisson(mean, N_DOCS)
        start = np.zeros(N_DOCS + 1, np.int64)
        np.cumsum(lens, out=start[1:])
        w = 1.0 / np.arange(1, vocab + 1)
        if f == 0:
            w[-16:] = 0.0
        cdf = np.cumsum(w) / w.sum()
        tok = np.searchsorted(cdf, rng.random(int(start[-1]))).astype(np.int64) + base
        doc = np.repeat(np.arange(N_DOCS), lens)
        docs.append(doc), terms.append(tok), poss.append(np.arange(int(start[-1])) - start[doc])
        if f == 1:
            continue
        last = lens.astype(np.int64) - 1

        def append(d, toks):   # one more value of each doc of d (distinct docs) holding toks
            d = np.asarray(d, np.int64)
            toks = np.broadcast_to(np.asarray(toks, np.int64), (len(d), np.shape(toks)[-1]))
            p = last[d][:, None] + pr.GAP + 1 + np.arange(toks.shape[1])
            docs.append(np.repeat(d, toks.shape[1])), terms.append(toks.ravel()), poss.append(p.ravel())
            last[d] = p[:, -1]
            return p

        def pick(n, fixed=()):
            fixed = np.array(sorted(fixed), np.int64)
            return np.concatenate([fixed, rng.choice(np.setdiff1d(np.arange(N_DOCS), fixed), n - len(fixed), replace=False)])
        da = pick(4096, EDGES)
        pa = append(da, A)
        docs.append(da[:500]), terms.append(np.full(500, STACK)), poss.append(pa[:500, 0])
        db = pick(4095, EDGES[::2])
        half = len(db) // 2
        append(db[:half], B)
        x = rng.integers(0, 50, (len(db) - half, 2))
        append(db[half:], np.stack([np.full(len(x), B[0]), x[:, 0], np.full(len(x), B[1]), x[:, 1], np.full(len(x), B[2])], 1))
        append(pick(1500), C8)
        hot = np.concatenate([HOT, rng.choice(np.setdiff1d(da, HOT), 18, replace=False)])
        append(hot[:10], np.tile(A, 299))   # with the planted value: tf 300
        append(hot[10:], np.tile(A, 254))   # tf 255
    term_field = np.array([0] * V0 + [1] * V1, np.int32)
    sh = pr.shard_from_token_arrays(N_DOCS, term_field, 2, np.concatenate(docs), np.concatenate(terms), np.concatenate(poss),
                                    live_docs=(rng.random(N_DOCS) > 0.05).astype(np.uint8))
    from nrtsearch_b200 import index as ix
    sh.doc_base = DOC_BASE
    sh.fields[1].norms = None
    n_vals = rng.integers(0, 4, N_DOCS)
    off = np.zeros(N_DOCS + 1, np.int64)
    np.cumsum(n_vals, out=off[1:])
    vals = rng.integers(0, 1000, int(off[-1]))
    vals = vals[np.lexsort((vals, np.repeat(np.arange(N_DOCS), n_vals)))].astype(np.int64)
    sh.columns, sh.column_has, sh.column_offsets = [ix.synth_int_column(N_DOCS), vals], [None, None], [None, off]
    return sh


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    sh = token_shard()
    g = GpuIndex(gpu_ctx, sh)
    yield sh, g
    g.close()


def T(t):
    return TermQuery(int(t))


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(T(c) if isinstance(c, (int, np.integer)) else c, o)
    return q


def match(*terms):
    return bq(*[(t, S) for t in terms])


def P(terms, slop=0, positions=None):
    return PhraseQuery([int(t) for t in terms], positions, slop)


def tree_queries():
    return [
        bq((match(3, 5), M), (PRICE, F)),                                             # match-in-bool
        DisjunctionMaxQuery([match(3, 9), match(V0 + 2, V0 + 7)], 0.0),               # multi_match
        bq((DisjunctionMaxQuery([match(3, 9), match(V0 + 2, V0 + 7)], 0.3), M), (MV, S)),
        bq((bq((2, S), (4, S), (6, S), msm=2), M), (8, S)),                           # inner msm
        bq((match(1, 2), F), (bq((3, S), (5, S)), N), (7, S)),                        # FILTER and MUST_NOT subtrees
        bq((bq((bq((bq((1, S), (2, S)), M), (3, S), (4, S)), S), (5, S)), M), (6, S), (7, S), (A[0], S)),   # depth 4, 8 slots
        bq((match(3, 4), S), (bq((3, M), (9, S)), S)),                                # a term repeated across branches
        bq((BoostQuery(PRICE, 2.0), S), (BoostQuery(MatchAllDocsQuery(), 0.5), S), (BoostQuery(MV, 1.5), S), (5, S)),
        match(A[0], 5, B[0]),                                                         # tf 255 / 300, row and no-row lists
    ]


def phrase_queries():
    dm = DisjunctionMaxQuery([P(A), P(C1), T(7)], 0.3)
    return [
        P(A), P(B), P(C8), P(C8[:5]), P(A, 1), P(B, 2), P([B[2], B[0]], 5), P(B, 101), P(C1, 2),
        P([B[2], B[1]]),                                                              # co-occur, never as the phrase
        bq((match(*B), M), (BoostQuery(P(B), 2.0), S)),
        bq((P(A), F), (11, S), (12, S)), bq((5, S), (9, S), (P(A), N)),
        bq((P(B, 2), M), (PRICE, F)),
        bq((bq((P(A), M), (4, S)), S), (bq((P(C8[:3]), F), (P(B[:2], 1), S)), S)),   # 8 slots
        dm, bq((dm, M), (PRICE, S)),
        BoostQuery(P(B), 3.0), bq((BoostQuery(P(A, 2), 0.5), S), (P(B), S), msm=1),
        P([A[0], STACK, A[1]], positions=[0, 0, 1]), P([STACK, A[1]]),
        P([A[0]]), P([]), bq((P([]), M), (3, S)),                                     # one term, no term, a root that cannot match
    ]


QUERIES = tree_queries() + phrase_queries()


@pytest.fixture(scope="module")
def reference(corpus):
    sh, _ = corpus
    leaves = pr.PhraseLeaves(sh, oracle.OracleIndex(sh), None, None)
    present, score = rr.evaluate_all(sh, QUERIES, leaves=leaves)
    return present, score, leaves


def hit_lists(present, n_hits, seed):
    """per query: half matching docs, half random docs around the shard, duplicates, docs outside it and the edge docs"""
    rng = np.random.default_rng(seed)
    nq = present.shape[0]
    docs = np.empty((nq, n_hits), np.int64)
    for q in range(nq):
        m = np.nonzero(present[q])[0]
        k = n_hits // 2 if len(m) else 0
        a = rng.choice(m, k, replace=len(m) < k) if k else np.zeros(0, np.int64)
        b = rng.integers(-20, N_DOCS + 20, n_hits - k)
        d = rng.permutation(np.concatenate([a, b]))
        if n_hits >= 64:
            d[:len(EDGES)] = EDGES
            d[len(EDGES):len(EDGES) + 3] = [-1, N_DOCS, -DOC_BASE]
            d[-5:] = d[len(EDGES) + 3:len(EDGES) + 8]   # duplicates
        docs[q] = d + DOC_BASE
    return docs.astype(np.int32)


def check_second_pass(got, want, what):
    gm, gs = got
    wm, ws = want
    bad = np.nonzero((gm != wm).any(1) | (gs.view(np.uint32) != ws.view(np.uint32)).any(1))[0]
    assert not len(bad), f"{what}: queries {bad.tolist()} differ, first at hit {np.nonzero(gm[bad[0]] != wm[bad[0]])[0][:5]}"


def test_the_shard_reaches_its_edges(corpus, reference):
    sh, _ = corpus
    present = reference[0]
    assert sh.df(A[0]) == sh.df(A[1]) == 4096 and sh.df(B[0]) == 4095 and sh.df(C8[0]) == 1500
    lst = sh.post_docs[sh.term_off[A[0]]:sh.term_off[A[0] + 1]]
    assert {0, 1023, 1024, 2047, N_DOCS - 1} <= set(lst.tolist())
    f = sh.post_freqs[sh.term_off[A[0]]:sh.term_off[A[0] + 1]]
    assert (f == 300).sum() == 10 and (f == 255).sum() == 10
    assert sh.df(3) * 64 >= N_DOCS and sh.df(2500) < 4096   # a plane term, a short list
    nq = len(QUERIES)
    assert present[len(tree_queries()) + 9].sum() == 0            # never as the phrase
    assert present[nq - 1].sum() == 0 and present[nq - 2].sum() == 0
    assert (present.sum(1) > 0).sum() >= nq - 3


@pytest.mark.parametrize("n_hits", [1, 1000, 4096])
def test_second_pass_equals_the_reference(corpus, reference, n_hits):
    sh, g = corpus
    present, score, _ = reference
    docs = hit_lists(present, n_hits, n_hits)
    rng = np.random.default_rng(n_hits + 1)
    counts = rng.integers(0, n_hits + 1, len(QUERIES)).astype(np.int32)
    counts[0], counts[1] = 0, n_hits
    s = GpuIndexSearcher(g)
    check_second_pass(s.score_docs_tree(QUERIES, docs, counts), rr.read_at_hits(sh, present, score, docs, counts), "counts")
    check_second_pass(s.score_docs_tree(QUERIES, docs), rr.read_at_hits(sh, present, score, docs), "counts NULL")
    if n_hits >= 1000:
        assert rr.read_at_hits(sh, present, score, docs)[0].sum() > len(QUERIES) * n_hits // 4


@pytest.mark.parametrize("weights", [(1.0, 4.0), (0.0, 1.0), (1.0, 0.0)])
def test_rescore_a_match_page_by_its_phrase(corpus, reference, weights):
    """QueryRescorer as users run it: the first-pass page of a match rescored by the phrase of its tokens"""
    sh, g = corpus
    s = GpuIndexSearcher(g)
    toks = [A, B, C8[:3], C1, [B[2], B[1]], [A[0], 7]]
    first = s.search_tree([match(*t) for t in toks], RelevanceCollector(1000, INT_MAX))
    rescore = [P(toks[0]), P(toks[1], 2), bq((P(toks[2]), S), (BoostQuery(P(C8[3:6], 1), 2.0), S)), P(toks[3], 1), P(toks[4]),
               DisjunctionMaxQuery([P(toks[5]), P(A, 1)], 0.3)]
    want_m, want_s = rr.score_docs(sh, rescore, first.docs, first.counts, leaves=reference[2])
    assert want_m.sum() > 2000
    for window in (1, 2, 40, 1001):
        d, sc, c = s.rescore_query_tree(rescore, first.docs, first.scores, first.counts, window, *weights)
        wd, ws, wc = rr.rescore(first.docs, first.scores, want_m, want_s, first.counts, window, *weights)
        assert np.array_equal(c, wc)
        for q in range(len(toks)):
            n = int(wc[q])
            assert np.array_equal(d[q, :n], wd[q, :n]), f"window {window} query {q}: docs"
            assert np.array_equal(sc[q, :n].view(np.uint32), ws[q, :n].view(np.uint32)), f"window {window} query {q}: scores"


def test_rescore_adversarial_hit_lists(corpus, reference):
    sh, g = corpus
    present, score, _ = reference
    docs = hit_lists(present, 4096, 7)
    first = np.random.default_rng(8).random(docs.shape).astype(np.float32) * 10
    counts = np.random.default_rng(9).integers(0, 4097, len(QUERIES)).astype(np.int32)
    counts[0], counts[1] = 0, 4096
    wm, ws = rr.read_at_hits(sh, present, score, docs, counts)
    s = GpuIndexSearcher(g)
    for window in (1, 40, 4096):
        d, sc, c = s.rescore_query_tree(QUERIES, docs, first, counts, window, 1.0, 4.0)
        wd, wsc, wc = rr.rescore(docs, first, wm, ws, counts, window, 1.0, 4.0)
        assert np.array_equal(c, wc)
        for q in range(len(QUERIES)):
            n = int(wc[q])
            assert np.array_equal(d[q, :n], wd[q, :n]) and np.array_equal(sc[q, :n].view(np.uint32), wsc[q, :n].view(np.uint32)), q


def test_each_query_scores_its_own_first_pass_page(corpus):
    """cross-engine: a tree query's top-1024 page from the window engine comes back all matched with the same floats"""
    _, g = corpus
    s = GpuIndexSearcher(g)
    page = s.search_tree(QUERIES, RelevanceCollector(1024, INT_MAX))
    m, sc = s.score_docs_tree(QUERIES, page.docs, page.counts)
    assert page.counts.sum() > 10_000
    for q in range(len(QUERIES)):
        n = int(page.counts[q])
        assert m[q, :n].all(), f"query {q}: a page hit does not match in the second pass"
        assert np.array_equal(sc[q, :n].view(np.uint32), page.scores[q, :n].view(np.uint32)), f"query {q}: scores differ"
        assert not m[q, n:].any()


FLAT = [bq((3, S), (5, S)), bq((2, M), (7, S), (PRICE, F)), match(1, 4, 8, A[0]), bq((MV, F), (6, S)), bq((B[0], M), (9, N))]


def test_flat_requests_are_the_flat_pair(corpus, reference):
    sh, g = corpus
    L = _native.gpu_lib()
    carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(FLAT, phrase_table=True)
    assert nn == 0 and n_ph == 0
    docs = hit_lists(reference[0][:nq], 1000, 11)
    counts = np.full(nq, 900, np.int32)
    outs = [(np.zeros(docs.shape, np.uint8), np.zeros(docs.shape, np.float32)) for _ in range(2)]
    assert L.nrtgpu_score_docs_tree(g.handle, carr, ncl, narr, 0, parr, 0, tarr, 0, qarr, nq, 1000, docs.ctypes.data,
                                    counts.ctypes.data, None, outs[0][0].ctypes.data, outs[0][1].ctypes.data) == 0
    assert L.nrtgpu_score_docs(g.handle, carr, ncl, qarr, nq, 1000, docs.ctypes.data, counts.ctypes.data, None,
                               outs[1][0].ctypes.data, outs[1][1].ctypes.data) == 0
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1].view(np.uint32), outs[1][1].view(np.uint32))
    assert outs[0][0].sum() > 1000
    first = np.random.default_rng(12).random(docs.shape).astype(np.float32)
    res = []
    for tree in (True, False):
        d, s_, oc = docs.copy(), first.copy(), np.zeros(nq, np.int32)
        if tree:
            rc = L.nrtgpu_rescore_query_tree(g.handle, carr, ncl, narr, 0, parr, 0, tarr, 0, qarr, nq, 1000, counts.ctypes.data, 40,
                                             1.0, 4.0, None, d.ctypes.data, s_.ctypes.data, oc.ctypes.data)
        else:
            rc = L.nrtgpu_rescore_query(g.handle, carr, ncl, qarr, nq, 1000, counts.ctypes.data, 40, 1.0, 4.0, None, d.ctypes.data,
                                        s_.ctypes.data, oc.ctypes.data)
        assert rc == 0
        res.append((d, s_, oc))
    for x, y in zip(*res):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
    # the Python wrappers: score_docs_tree of a flat batch is score_docs
    s = GpuIndexSearcher(g)
    a, b = s.score_docs_tree(FLAT, docs, counts), s.score_docs(FLAT, docs, counts)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def test_mixed_flat_and_tree_batch(corpus, reference):
    sh, g = corpus
    qs = FLAT + [QUERIES[0], QUERIES[len(tree_queries())], QUERIES[-4]]
    present, score = rr.evaluate_all(sh, qs, leaves=reference[2])
    docs = hit_lists(present, 1000, 13)
    check_second_pass(GpuIndexSearcher(g).score_docs_tree(qs, docs), rr.read_at_hits(sh, present, score, docs), "mixed")


def test_three_leaves_with_doc_base_equal_the_single_image(gpu_ctx, corpus, reference):
    sh, g = corpus
    docs = hit_lists(reference[0], 1000, 17)
    want = GpuIndexSearcher(g).score_docs_tree(QUERIES, docs)
    cuts = [0, 100_000, 262_147, N_DOCS]
    m, s = np.zeros(docs.shape, np.uint8), np.zeros(docs.shape, np.float32)
    for a, b in zip(cuts, cuts[1:]):
        leaf = GpuIndex(gpu_ctx, sh.doc_range(a, b))
        try:
            lm, ls = GpuIndexSearcher(leaf).score_docs_tree(QUERIES, docs)
        finally:
            leaf.close()
        assert not (m & lm).any()
        m |= lm
        s = np.where(lm != 0, ls, s)
    check_second_pass((m, s), want, "three leaves")
    check_second_pass((m, s), rr.read_at_hits(sh, reference[0], reference[1], docs), "three leaves vs reference")


def test_follows_live_docs_and_stats(gpu_ctx, corpus):
    sh, _ = corpus
    small = sh.doc_range(0, 150_000)
    g = GpuIndex(gpu_ctx, small)
    try:
        qs = [P(A), P(B, 2), bq((match(*B), M), (BoostQuery(P(B), 2.0), S)), QUERIES[1], QUERIES[5]]
        rng = np.random.default_rng(3)
        small.live_docs = (rng.random(small.n_docs) > 0.2).astype(np.uint8)
        g.set_live_docs(small.live_docs)
        small.term_df = (small.term_df * 3 + 1).astype(np.int64)
        for f in small.fields:
            f.doc_count, f.sum_total_term_freq = f.doc_count * 4, f.sum_total_term_freq * 5
        g.update_stats(small.term_df, [f.doc_count for f in small.fields], [f.sum_total_term_freq for f in small.fields])
        present, score = rr.evaluate_all(small, qs)
        docs = hit_lists(present, 1000, 19)
        check_second_pass(GpuIndexSearcher(g).score_docs_tree(qs, docs), rr.read_at_hits(small, present, score, docs), "refresh")
    finally:
        g.close()


def _score(g, a, docs=None, n_hits=4, counts=None):
    nq = a[9]
    d = np.full((max(nq, 1), n_hits), DOC_BASE, np.int32) if docs is None else docs
    m, s = np.zeros(d.shape, np.uint8), np.zeros(d.shape, np.float32)
    return _native.gpu_lib().nrtgpu_score_docs_tree(g.handle, *a[:9], nq, n_hits, d.ctypes.data,
                                                    None if counts is None else counts.ctypes.data, None, m.ctypes.data, s.ctypes.data)


def _rescore(g, a, n_hits=4, window=2, counts=None):
    nq = a[9]
    d, s = np.full((nq, n_hits), DOC_BASE, np.int32), np.ones((nq, n_hits), np.float32)
    c = np.full(nq, n_hits, np.int32) if counts is None else counts
    return _native.gpu_lib().nrtgpu_rescore_query_tree(g.handle, *a[:9], nq, n_hits, c.ctypes.data, window, 1.0, 2.0, None,
                                                       d.ctypes.data, s.ctypes.data, None)


@pytest.mark.parametrize("case", range(len(INVALID_PHRASES)))
def test_invalid_phrases(corpus, case):
    _, g = corpus
    clauses, phrases, terms, msg = INVALID_PHRASES[case]
    if msg == "same field":
        terms = [(1, 0), (V0 + 1, 1)]
    if msg == "phrase term id out of range":
        terms = [(1, 0), (10**8, 1)]
    a = _arrays(clauses, phrases, terms)
    for call in (_score, _rescore):
        assert call(g, a) == 1 and msg in _native.gpu_lib().nrtgpu_last_error().decode(), call.__name__


def test_invalid_and_unsupported_status(gpu_ctx, corpus):
    sh, g = corpus
    L = _native.gpu_lib()
    a = compile_tree([P(A), QUERIES[5]], phrase_table=True)
    assert _score(g, a, n_hits=0) == 1 and "bad argument" in L.nrtgpu_last_error().decode()
    assert L.nrtgpu_score_docs_tree(g.handle, *a[:9], a[9], 4, None, None, None, None, None) == 1
    assert _rescore(g, a, window=0) == 1
    assert _rescore(g, a, counts=np.array([5, 1], np.int32)) == 1 and "counts out of range" in L.nrtgpu_last_error().decode()
    assert _rescore(g, a, n_hits=4097) == 3 and "4096" in L.nrtgpu_last_error().decode()
    assert _score(g, a[:2] + (None, -1) + a[4:]) == 1
    # tree limits and the phrase refusals of nrtgpu_search_tree_phrases
    for qs in ([P([B[0], B[0]], 1)], [bq((P(C8[:5]), M), (1, S), (2, S), (3, S), (4, S))], [bq(*[(P([]), S)] * 30, (P(B), S))],
               [bq((bq((bq((bq((bq((1, S), (2, S)), M), (3, S)), M), (4, S)), M), (5, S)), M))]):
        b = compile_tree(qs, phrase_table=True)
        assert _score(g, b) == 3 and _rescore(g, b) == 3, L.nrtgpu_last_error()
    with pytest.raises(NrtGpuUnsupported):
        GpuIndexSearcher(g).score_docs_tree([P([A[0], A[0]], 2)], np.zeros((1, 4), np.int32))
    # an image without positions
    small = sh.doc_range(0, 50_000)
    small.post_positions = None
    g2 = GpuIndex(gpu_ctx, small)
    try:
        for call in (_score, _rescore):
            assert call(g2, compile_tree([P(A)], phrase_table=True)) == 1 and "without position data" in L.nrtgpu_last_error().decode()
        assert _score(g2, compile_tree([QUERIES[5]], phrase_table=True)) == 0   # a tree without phrases needs no positions
    finally:
        g2.close()
    # the flat pair keeps refusing node and phrase clauses
    for qs in ([bq((P(A), M), (3, S))], [QUERIES[5]]):
        c = compile_tree(qs, phrase_table=True)
        d, m, s = np.full((1, 4), DOC_BASE, np.int32), np.zeros((1, 4), np.uint8), np.zeros((1, 4), np.float32)
        assert L.nrtgpu_score_docs(g.handle, c[0], c[1], c[8], c[9], 4, d.ctypes.data, None, None, m.ctypes.data, s.ctypes.data) == 1
        assert "bad clause kind" in L.nrtgpu_last_error().decode()
        assert L.nrtgpu_rescore_query(g.handle, c[0], c[1], c[8], c[9], 4, None, 2, 1.0, 1.0, None, d.ctypes.data, s.ctypes.data,
                                      None) == 1
        assert "bad clause kind" in L.nrtgpu_last_error().decode()
    with pytest.raises(NrtGpuError):
        GpuIndexSearcher(g).score_docs([P(A)], np.zeros((1, 4), np.int32))
