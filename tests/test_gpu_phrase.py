"""Phrase leaves on the GPU (nrtgpu_search_tree_phrases, the tree instantiation of bool_window_kernel) against
tests/phrase_reference.py, bit for bit: docs, scores, counts and totalHits at top_k 1, 40, 100 and 1024, in COMPLETE mode and
at totalHitsThreshold 1000.

The shard: 1.25M docs built from token sequences (two text fields with positions, a third of field 0's docs two-valued with a
position increment gap of 100), 5% deletes and a price column. Reserved field-0 terms, never drawn at random, carry planted
phrases: 2-, 3-, 8- and 3-fold repeated-term phrases in thousands of docs, on both sides of window (16,384) and slice
(1,048,576) edges and at n_docs - 1; docs where a phrase term has tf 300; and a stacked term at the position of another."""
import numpy as np
import pytest

import phrase_reference as pr
from nrtsearch_b200 import NrtGpuError, NrtGpuUnsupported, _native
from nrtsearch_b200._native import CollectionTimeoutException
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, GpuIndex, GpuIndexSearcher, Occur, PhraseQuery,
                                   RangeQuery, RelevanceCollector, ScoreDoc, TermQuery, compile_queries, compile_tree)
from test_phrase_plan import INVALID_PHRASES, _arrays

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
N_DOCS = 1_250_000
V0, V1 = 5000, 4000
WIDE_SLICE = 64 * 16384
S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
R = [V0 - 16 + i for i in range(16)]            # reserved field-0 terms: planted only
A, B, C8, REP = R[0:2], R[2:5], R[5:13], [R[14]] * 3
STACK = R[13]                                   # stacked at the position of A's first term in some docs
EDGES = sorted({d for e in (0, 16384, 2 * 16384, WIDE_SLICE, WIDE_SLICE + 16384, N_DOCS) for d in (e - 2, e - 1, e, e + 1)
                if 0 <= d < N_DOCS})
PRICE = RangeQuery(0, 100_000, 800_000)


def token_shard():
    rng = np.random.default_rng(41)
    docs, terms, poss = [], [], []
    for f, (lo, mean, vocab, base) in enumerate(((4, 6.0, V0, 0), (2, 4.0, V1, V0))):
        lens = lo + rng.poisson(mean, N_DOCS)
        start = np.zeros(N_DOCS + 1, np.int64)
        np.cumsum(lens, out=start[1:])
        w = 1.0 / np.arange(1, vocab + 1) ** 1.0
        if f == 0:
            w[-16:] = 0.0
        cdf = np.cumsum(w) / w.sum()
        tok = np.searchsorted(cdf, rng.random(int(start[-1]))).astype(np.int64) + base
        doc = np.repeat(np.arange(N_DOCS), lens)
        pos = np.arange(int(start[-1])) - start[doc]
        if f == 0:
            two = rng.random(N_DOCS) < 0.33                      # two values: the second starts after the gap
            split = rng.integers(1, lens)
            pos = pos + np.where(two[doc] & (pos >= split[doc]), pr.GAP, 0)

            def plant(phrase, n, fixed=()):
                cand = np.nonzero(lens >= len(phrase))[0]
                d = np.concatenate([rng.choice(cand, n, replace=False), np.array(fixed, np.int64)])
                s = np.where(np.isin(d, fixed), 0, rng.integers(0, lens[d] - len(phrase) + 1))
                tok[start[d][:, None] + s[:, None] + np.arange(len(phrase))] = phrase
                return d, s
            plant(B, 3000, EDGES[::2])
            plant(C8, 1500, EDGES[1::3])
            plant(REP, 800)
            da, sa = plant(A, 6000, EDGES)
            extra_d, extra_t, extra_p = [], [], []
            st = da[:500]                                         # STACK at the position of A's first term
            extra_d.append(st), extra_t.append(np.full(len(st), STACK)), extra_p.append(pos[start[st] + sa[:500]])
            hot = np.concatenate([rng.choice(N_DOCS, 20, replace=False), [N_DOCS - 1, WIDE_SLICE, 16383]])
            for d in hot:                                         # a third value: "A0 A1" 300 times (tf 300)
                extra_d.append(np.full(600, d)), extra_t.append(np.tile(A, 300))
                extra_p.append(pos[start[d + 1] - 1] + pr.GAP + 1 + np.arange(600))
            doc = np.concatenate([doc] + extra_d)
            tok = np.concatenate([tok] + extra_t)
            pos = np.concatenate([pos] + extra_p)
        docs.append(doc), terms.append(tok), poss.append(pos)
    term_field = np.array([0] * V0 + [1] * V1, np.int32)
    sh = pr.shard_from_token_arrays(N_DOCS, term_field, 2, np.concatenate(docs), np.concatenate(terms), np.concatenate(poss),
                                    live_docs=(rng.random(N_DOCS) > 0.05).astype(np.uint8))
    from nrtsearch_b200 import index as ix
    sh.columns, sh.column_has = [ix.synth_int_column(N_DOCS)], [None]
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


def phrase_queries():
    c1 = [V0 + 3, V0 + 5]                                           # a common field-1 bigram
    dm = DisjunctionMaxQuery([P(A), P(c1), T(7)], 0.3)
    return [
        P(A), P(B), P(C8), P(C8[:5]), P(C8[2:8]), P(A + [B[0]]),
        P(A, 1), P(B, 2), P([B[2], B[0]], 5), P(B, 101), P(c1, 2),
        P([B[2], B[1]]),                                            # every term occurs, never this phrase
        bq((match(*B), M), (BoostQuery(P(B), 2.0), S)),            # match + phrase boost
        bq((match(*c1), M), (BoostQuery(P(c1), 2.0), S)),
        bq((P(A), F), (11, S), (12, S)), bq((5, S), (9, S), (P(A), N)),
        bq((P(B), M), (PRICE, F)), bq((bq((P(B), S), (3, S)), M), (PRICE, F)),
        bq((bq((P(A), M), (4, S)), S), (bq((P(C8[:3]), F), (P(B[:2], 1), S)), S)),   # 8 slots
        bq((bq((3, S), (7, S), (P(A), N)), M), (P(c1), N), (PRICE, F)),
        dm, bq((dm, M), (PRICE, S)),
        BoostQuery(P(B), 3.0), bq((BoostQuery(P(A, 2), 0.5), S), (P(B), S), msm=1),
        P([A[0], STACK, A[1]], positions=[0, 0, 1]), P([STACK, A[1]]), P(REP[:2]), P(REP), P([STACK])
    ]


@pytest.fixture(scope="module")
def batch(corpus):
    sh, _ = corpus
    qs = phrase_queries()
    return qs, pr.search(sh, qs, 1024)


def check(res, want, k, what=""):
    for q in range(len(res.counts)):
        n = min(int(want[2][q]), k)
        assert res.counts[q] == n, f"{what} query {q}: counts {res.counts[q]} vs {n}"
        assert np.array_equal(res.docs[q, :n], want[0][q, :n]), f"{what} query {q}: docs differ"
        assert np.array_equal(res.scores[q, :n].view(np.uint32), want[1][q, :n].view(np.uint32)), f"{what} query {q}: scores differ"
    assert np.array_equal(res.total_hits, want[3]), f"{what}: totalHits differ"
    assert not res.relation.any()


def test_the_shard_reaches_its_edges(corpus, batch):
    sh, _ = corpus
    qs, want = batch
    assert (want[3][:4] > 1000).all() and want[3][11] == 0 and (want[3] > 0).sum() >= len(qs) - 1
    for q in (0, 1):   # planted A and B are found on both sides of the edges and at n_docs - 1
        got = set(want[0][q, :want[2][q]].tolist())
        assert any(e in got for e in EDGES) or want[3][q] > 1024
    assert sh.post_freqs.max() >= 300


@pytest.mark.parametrize("k", [1, 40, 100, 1024])
@pytest.mark.parametrize("threshold", [INT_MAX, 1000])
def test_phrases_equal_the_reference(corpus, batch, k, threshold):
    _, g = corpus
    qs, want = batch
    res = GpuIndexSearcher(g).search_tree(qs, RelevanceCollector(k, threshold))
    check(res, want, k, f"k={k} thr={threshold}")


def test_edge_docs(corpus):
    """a phrase found only at the window / slice edges and at n_docs - 1 (the docs that hold A at position 0 and tf-300 A)"""
    sh, g = corpus
    qs = [bq((P(A), M), (RangeQuery(0, -(2**63), 2**63 - 1), F))]
    want = pr.search(sh, qs, 1024)
    res = GpuIndexSearcher(g).search_tree(qs, RelevanceCollector(1024, INT_MAX))
    check(res, want, 1024, "edges")
    live_edges = [e for e in EDGES if sh.live_docs[e]]
    assert set(live_edges) <= set(want[0][0, :want[2][0]].tolist()) or want[3][0] > 1024


def test_search_after_pages(corpus, batch):
    _, g = corpus
    qs, want = batch
    s = GpuIndexSearcher(g)
    k = 40
    p1 = s.search_tree(qs, RelevanceCollector(k, INT_MAX))
    after = [ScoreDoc(int(p1.docs[q, k - 1]), float(p1.scores[q, k - 1])) if p1.counts[q] == k else None for q in range(len(qs))]
    p2 = s.search_tree(qs, RelevanceCollector(k, INT_MAX), search_after=after)
    assert sum(a is not None for a in after) > len(qs) // 2
    for q in range(len(qs)):
        if after[q] is None:
            continue
        n = int(p2.counts[q])
        assert n == min(k, int(want[3][q]) - k)
        assert np.array_equal(p2.docs[q, :n], want[0][q, k:k + n]), f"query {q}: page 2 docs"
        assert np.array_equal(p2.scores[q, :n].view(np.uint32), want[1][q, k:k + n].view(np.uint32)), f"query {q}: page 2 scores"


def test_deadline_and_terminate_after(corpus, batch):
    _, g = corpus
    qs, want = batch
    s = GpuIndexSearcher(g)
    late = s.search_tree(qs, RelevanceCollector(10, INT_MAX, timeout_sec=0.5, elapsed_sec=1.0))
    assert late.hit_timeout.all() and late.relation.all() and not late.counts.any()
    with pytest.raises(CollectionTimeoutException):
        s.search_tree(qs, RelevanceCollector(10, INT_MAX, timeout_sec=0.5, elapsed_sec=1.0, disallow_partial_results=True))
    T_, R_ = 500, 800
    res = s.search_tree(qs, RelevanceCollector(10, INT_MAX, terminate_after=T_, terminate_after_max_recall_count=R_))
    term = want[3] > T_
    assert np.array_equal(res.terminated_early != 0, term)
    assert np.array_equal(res.total_hits, np.where(term, np.minimum(want[3], R_), want[3]))
    for q in range(len(qs)):
        n = int(res.counts[q])
        assert np.array_equal(res.docs[q, :n], want[0][q, :n]) and np.array_equal(res.scores[q, :n], want[1][q, :n])


def test_three_leaves_with_doc_base_equal_the_whole_reader(gpu_ctx, corpus, batch):
    import torch
    from nrtsearch_b200.shards import PackedGather
    sh, _ = corpus
    qs, want = batch
    cuts = [0, 400_000, WIDE_SLICE + 3, N_DOCS]
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    nq, k = len(qs), 100
    dev = torch.device("cuda", 0)
    pg = PackedGather(nq, k, len(leaves), dev)
    try:
        recs = []
        for g in leaves:
            b = GpuIndexSearcher(g).prepare_tree(qs, RelevanceCollector(k, INT_MAX))
            rec = torch.zeros(pg.words, dtype=torch.int32, device=dev)
            b.bind_packed(rec.data_ptr()); b.run(); torch.cuda.synchronize(); b.close()
            recs.append(rec)
        pg.all.copy_(torch.cat(recs))
        pg.merge_on_device(gpu_ctx, 0)
        torch.cuda.synchronize()
        d, s_, c, flags, tot = pg.unpack()
        for q in range(nq):
            n = min(int(want[2][q]), k)
            assert c[q] == n and np.array_equal(d[q, :n], want[0][q, :n]), f"query {q}: docs"
            assert np.array_equal(s_[q, :n].view(np.uint32), want[1][q, :n].view(np.uint32)), f"query {q}: scores"
        assert np.array_equal(tot, want[3]) and not flags.any()
    finally:
        for g in leaves:
            g.close()


def _outs(nq, k):
    return [np.zeros(nq * k, np.int32), np.zeros(nq * k, np.float32), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
            np.zeros(nq, np.uint8), np.zeros(nq, np.uint8), np.zeros(nq, np.uint8)]


def _call_phrases(g, a, k=10):
    out = _outs(a[9], k)
    rc = _native.gpu_lib().nrtgpu_search_tree_phrases(g.handle, *a[:9], a[9], k, INT_MAX, 0, None, None, *[o.ctypes.data for o in out])
    return rc, out


def test_no_phrases_is_search_tree(corpus):
    _, g = corpus
    qs = [bq((match(3, 5), M), (PRICE, F)), bq((DisjunctionMaxQuery([match(3, 9), match(V0 + 2, V0 + 7)], 0.2), M)), match(4, 8, 15)]
    for threshold in (INT_MAX, 1000):
        carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(qs, phrase_table=True)
        assert n_ph == 0
        a, b = _outs(nq, 50), _outs(nq, 50)
        L = _native.gpu_lib()
        assert L.nrtgpu_search_tree_phrases(g.handle, carr, ncl, narr, nn, parr, 0, tarr, 0, qarr, nq, 50, threshold, 0, None, None,
                                            *[o.ctypes.data for o in a]) == 0
        assert L.nrtgpu_search_tree(g.handle, carr, ncl, narr, nn, qarr, nq, 50, threshold, 0, None, None, *[o.ctypes.data for o in b]) == 0
        for x, y in zip(a, b):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


def test_positions_survive_live_docs_and_stats(gpu_ctx, corpus):
    sh, _ = corpus
    small = sh.doc_range(0, 300_000)
    g = GpuIndex(gpu_ctx, small)
    try:
        qs = [P(A), P(B, 2), bq((match(*B), M), (BoostQuery(P(B), 2.0), S))]
        rng = np.random.default_rng(3)
        small.live_docs = (rng.random(small.n_docs) > 0.2).astype(np.uint8)
        g.set_live_docs(small.live_docs)
        small.term_df = (small.term_df * 3 + 1).astype(np.int64)
        for f in small.fields:
            f.doc_count, f.sum_total_term_freq = f.doc_count * 4, f.sum_total_term_freq * 5
        g.update_stats(small.term_df, [f.doc_count for f in small.fields], [f.sum_total_term_freq for f in small.fields])
        want = pr.search(small, qs, 100)
        check(GpuIndexSearcher(g).search_tree(qs, RelevanceCollector(100, INT_MAX)), want, 100, "after refresh")
    finally:
        g.close()


def test_add_positions_refusals_replace_and_device_bytes(gpu_ctx, corpus):
    sh, _ = corpus
    small = sh.doc_range(0, 100_000)
    pos = small.post_positions
    small.post_positions = None
    g = GpuIndex(gpu_ctx, small)
    L = _native.gpu_lib()
    try:
        before = g.device_bytes
        rc, _ = _call_phrases(g, compile_tree([P(A)], phrase_table=True))
        assert rc == 1 and "without position data" in L.nrtgpu_last_error().decode()
        for bad, msg in ((pos[:-1], "sum of the postings' freqs"), (np.where(np.arange(len(pos)) == 5, -1, pos), "negative"),
                         (pos[::-1].copy(), "descend")):
            with pytest.raises(NrtGpuError, match=msg):
                g.add_positions(bad)
        assert g.device_bytes == before
        g.add_positions(pos)
        n_terms, P_ = small.n_terms, len(small.post_docs)
        assert g.device_bytes - before == 4 * len(pos) + 4 * P_ + 8 * (n_terms + 1)
        g.add_positions(pos)   # replaces
        assert g.device_bytes - before == 4 * len(pos) + 4 * P_ + 8 * (n_terms + 1)
        small.post_positions = pos
        qs = [P(A), P(B, 1), P(C8)]
        check(GpuIndexSearcher(g).search_tree(qs, RelevanceCollector(100, INT_MAX)), pr.search(small, qs, 100), 100, "replaced")
    finally:
        g.close()


@pytest.mark.parametrize("case", range(len(INVALID_PHRASES)))
def test_invalid_status(corpus, case):
    _, g = corpus
    clauses, phrases, terms, msg = INVALID_PHRASES[case]
    if msg == "same field":
        terms = [(1, 0), (V0 + 1, 1)]
    if msg == "phrase term id out of range":
        terms = [(1, 0), (10**8, 1)]
    rc, _ = _call_phrases(g, _arrays(clauses, phrases, terms))
    assert rc == 1 and msg in _native.gpu_lib().nrtgpu_last_error().decode()


def test_unsupported_status_and_other_entry_points(corpus):
    _, g = corpus
    L = _native.gpu_lib()
    cases = [[P([B[0], B[0]], 1)], [bq((P(C8[:5]), M), (1, S), (2, S), (3, S), (4, S))],
             [bq(*[(P([]), S)] * 30, (P(B), S))]]
    for qs in cases:
        rc, _ = _call_phrases(g, compile_tree(qs, phrase_table=True))
        assert rc == 3, L.nrtgpu_last_error()
    rc, _ = _call_phrases(g, compile_tree([P(A)], phrase_table=True), k=1025)
    assert rc == 3
    with pytest.raises(NrtGpuUnsupported):
        GpuIndexSearcher(g).search_tree([P(B, 1), P([A[0], A[0]], 2)], RelevanceCollector(10, INT_MAX))
    # nrtgpu_search_tree and the flat entry points keep refusing kind 4
    carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree([bq((P(A), M), (match(1, 2), M))], phrase_table=True)
    out = _outs(nq, 1)
    assert L.nrtgpu_search_tree(g.handle, carr, ncl, narr, nn, qarr, nq, 1, INT_MAX, 0, None, None, *[o.ctypes.data for o in out]) == 1
    assert "bad clause kind" in L.nrtgpu_last_error().decode()
    flat = compile_tree([bq((P(A), M), (3, S))], phrase_table=True)
    o64 = np.zeros(16, np.int64)
    assert L.nrtgpu_search_bool(g.handle, flat[0], flat[1], flat[8], flat[9], 1, INT_MAX, 0, None, *[o64.ctypes.data] * 5) == 1
    assert "bad clause kind" in L.nrtgpu_last_error().decode()
    with pytest.raises(NrtGpuError):
        compile_queries([P(A)])
