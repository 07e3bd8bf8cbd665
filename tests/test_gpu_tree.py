"""Query trees on the GPU (nrtgpu_search_tree, the tree instantiation of bool_window_kernel) against tests/tree_reference.py,
bit for bit: docs, scores and totalHits at top_k 1, 40, 100 and 1024, in COMPLETE mode and at totalHitsThreshold 1000.

The shard: 1.25M docs (two 1,048,576-doc slices of the window engine) with two text fields, 5% deletes, a single-valued and
a multi-valued int column, and an appended term whose postings sit on both sides of window (16,384-doc) and slice edges."""
import numpy as np
import pytest

import tree_reference as tr
from nrtsearch_b200 import NrtGpuError, NrtGpuUnsupported, _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200._native import CollectionTimeoutException
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, GpuIndex, GpuIndexSearcher, MatchAllDocsQuery,
                                   Occur, RangeQuery, RelevanceCollector, ScoreDoc, TermQuery, compile_queries, compile_tree)
from test_tree_plan import INVALID_TREES

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
N_DOCS = 1_250_000
V = 20_000                      # vocabulary of each field
WIDE_SLICE = 64 * 16384
S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
EDGES = sorted({d for e in (0, 16384, 2 * 16384, WIDE_SLICE, WIDE_SLICE + 16384, N_DOCS) for d in (e - 2, e - 1, e, e + 1)
                if 0 <= d < N_DOCS})


def two_field_shard():
    """field 0: terms 0..V-1, field 1: terms V..2V-1, term 2V: the edge term (field 0); column 0 single-valued in
    [0, 1M), column 1 multi-valued (0..3 values in [0, 1000) per doc); 5% of the docs deleted"""
    a = ix.synth_text_shard(N_DOCS, V, min_len=4, poisson_mean=8.0)
    b = ix.synth_text_shard(N_DOCS, V, seed=ix.SEED_CORPUS + 7, min_len=2, poisson_mean=4.0)
    edge = np.array(EDGES, np.int32)
    off = np.concatenate([a.term_off, a.term_off[-1] + b.term_off[1:], [a.term_off[-1] + b.term_off[-1] + len(edge)]])
    docs = np.concatenate([a.post_docs, b.post_docs, edge])
    freqs = np.concatenate([a.post_freqs, b.post_freqs, np.full(len(edge), 2, np.int32)])
    fa = a.fields[0]
    fa.sum_total_term_freq += 2 * len(edge)
    sh = ix.HostShard(n_docs=N_DOCS, doc_base=0, term_off=off.astype(np.int64), post_docs=docs, post_freqs=freqs,
                      fields=[fa, b.fields[0]], term_field=np.array([0] * V + [1] * V + [0], np.int32))
    rng = np.random.default_rng(23)
    cnt = rng.integers(0, 4, N_DOCS)
    moff = np.zeros(N_DOCS + 1, np.int64)
    np.cumsum(cnt, out=moff[1:])
    vals = rng.integers(0, 1000, int(moff[-1])).astype(np.int64)
    vals = vals[np.lexsort((vals, np.repeat(np.arange(N_DOCS), cnt)))]
    sh.columns = [ix.synth_int_column(N_DOCS), vals]
    sh.column_has = [None, None]
    sh.column_offsets = [None, moff]
    sh.live_docs = (rng.random(N_DOCS) > 0.05).astype(np.uint8)
    sh.term_df = np.diff(sh.term_off).astype(np.int64)
    return sh


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    sh = two_field_shard()
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
    """a `match` of several tokens: BooleanQuery of SHOULD terms (QueryNodeMapper.getMatchQuery)"""
    return bq(*[(t, S) for t in terms])


PRICE = RangeQuery(0, 100_000, 800_000)
MV = RangeQuery(1, 200, 260)
EDGE = 2 * V


def shapes(t, u, tie):
    """every tree shape of the suite for field-0 terms t[0..5] and field-1 terms u[0..1]"""
    mm = DisjunctionMaxQuery([match(t[0], t[1]), match(u[0], u[1])], tie)
    return [
        bq((match(t[0], t[1]), M), (PRICE, F)),                                            # match in bool + range
        bq((match(t[0], t[1]), M), (match(t[2], t[3]), M)),                                # two matches
        bq((mm, M), (PRICE, F), (t[4], N)),                                                # multi_match under bool
        bq((bq((t[0], S), (t[1], S), (t[2], S), msm=2), M), (t[3], S)),                   # inner msm 2 of 3
        bq((t[0], S), (t[1], S), (match(t[2], t[3]), F), (bq((t[4], M), (MV, M)), N)),    # FILTER and MUST_NOT subtrees
        bq((bq((t[0], M), (t[1], M)), S), (match(t[2], t[3]), S), (t[4], S), msm=2),       # SHOULD subtrees, outer msm
        bq((bq((t[0], S), (bq((t[1], M), (match(t[2], t[3]), S)), S)), M), (match(t[4], t[5]), S), (u[0], S), (u[1], S)),  # depth 4, 8 leaves
        bq((bq((t[0], M), (t[1], S)), S), (bq((t[0], M), (t[2], S)), S)),                  # a term repeated across branches
        bq((BoostQuery(match(t[0], t[1]), 2.0), S), (BoostQuery(PRICE, 0.5), S), (BoostQuery(MatchAllDocsQuery(), 0.25), M)),
        BoostQuery(bq((BoostQuery(mm, 1.5), M), (BoostQuery(MV, 3.0), S)), 0.75),          # boosts around nodes
        bq((bq((t[0], S), (MV, S)), M), (PRICE, S)),                                       # dense driver
        bq((match(EDGE, t[0]), M), (bq((EDGE, S), (u[0], S)), S)),                          # the edge term
        mm,                                                                                # a dismax at the root
    ]


@pytest.fixture(scope="module")
def batch(corpus):
    sh, _ = corpus
    t = ix.synth_query_terms(8, 6, V, log10_lo=1.0, log10_hi=3.6)
    u = ix.synth_query_terms(8, 2, V, seed=ix.SEED_QUERIES + 1, log10_lo=1.0, log10_hi=3.3) + V
    qs = []
    for i in range(4):
        qs += shapes(t[i], u[i], 0.0 if i % 2 == 0 else 0.3)
    want = tr.search(sh, qs, 1024)
    return qs, want


def check(res, want, k, what=""):
    for q in range(len(res.counts)):
        n = min(int(want[2][q]), k)
        assert res.counts[q] == n, f"{what} query {q}: counts {res.counts[q]} vs {n}"
        assert np.array_equal(res.docs[q, :n], want[0][q, :n]), f"{what} query {q}: docs differ"
        assert np.array_equal(res.scores[q, :n].view(np.uint32), want[1][q, :n].view(np.uint32)), f"{what} query {q}: scores differ"
    assert np.array_equal(res.total_hits, want[3]), f"{what}: totalHits differ"
    assert not res.relation.any(), f"{what}: the window engine counts every hit"


@pytest.mark.parametrize("k", [1, 40, 100, 1024])
@pytest.mark.parametrize("threshold", [INT_MAX, 1000])
def test_trees_equal_the_reference(corpus, batch, k, threshold):
    _, g = corpus
    qs, want = batch
    assert (want[3] > 0).sum() > len(qs) * 3 // 4 and (want[3] > 1024).any()
    res = GpuIndexSearcher(g).search_tree(qs, RelevanceCollector(k, threshold))
    check(res, want, k, f"k={k} thr={threshold}")


def test_tree_batches_are_wide(corpus, batch):
    _, g = corpus
    qs, want = batch
    b = GpuIndexSearcher(g).prepare_tree(qs, RelevanceCollector(10, 1000))
    try:
        assert b.stats()["work_items"] == len(qs) * -(-N_DOCS // WIDE_SLICE)
    finally:
        b.close()


def test_search_after_pages(corpus, batch):
    _, g = corpus
    qs, want = batch
    s = GpuIndexSearcher(g)
    k = 40
    p1 = s.search_tree(qs, RelevanceCollector(k, INT_MAX))
    after = [ScoreDoc(int(p1.docs[q, k - 1]), float(p1.scores[q, k - 1])) if p1.counts[q] == k else None for q in range(len(qs))]
    p2 = s.search_tree(qs, RelevanceCollector(k, INT_MAX), search_after=after)
    for q in range(len(qs)):
        if after[q] is None:
            continue
        n = int(p2.counts[q])
        assert n == min(k, int(want[3][q]) - k), f"query {q}: page 2 holds {n} hits"
        assert np.array_equal(p2.docs[q, :n], want[0][q, k:k + n]), f"query {q}: page 2 docs"
        assert np.array_equal(p2.scores[q, :n].view(np.uint32), want[1][q, k:k + n].view(np.uint32)), f"query {q}: page 2 scores"
        assert p2.total_hits[q] == want[3][q]


def test_deadline_and_terminate_after(corpus, batch):
    _, g = corpus
    qs, want = batch
    s = GpuIndexSearcher(g)
    late = s.search_tree(qs, RelevanceCollector(10, INT_MAX, timeout_sec=0.5, elapsed_sec=1.0))
    assert late.hit_timeout.all() and late.relation.all() and not late.counts.any()
    with pytest.raises(CollectionTimeoutException, match="Search collection exceeded timeout of"):
        s.search_tree(qs, RelevanceCollector(10, INT_MAX, timeout_sec=0.5, elapsed_sec=1.0, disallow_partial_results=True))
    ok = s.search_tree(qs, RelevanceCollector(10, INT_MAX, timeout_sec=120.0))
    check(ok, want, 10, "generous deadline")
    T_, R = 500, 800
    res = s.search_tree(qs, RelevanceCollector(10, INT_MAX, terminate_after=T_, terminate_after_max_recall_count=R))
    term = want[3] > T_
    assert np.array_equal(res.terminated_early != 0, term) and np.array_equal(res.relation != 0, term)
    assert np.array_equal(res.total_hits, np.where(term, np.minimum(want[3], R), want[3]))
    for q in range(len(qs)):
        n = int(res.counts[q])
        assert np.array_equal(res.docs[q, :n], want[0][q, :n]) and np.array_equal(res.scores[q, :n], want[1][q, :n])


def flat_queries(n):
    t = ix.synth_query_terms(n, 3, V, seed=ix.SEED_QUERIES + 2, log10_lo=1.0, log10_hi=3.5)
    out = []
    for i, x in enumerate(t):
        out.append(match(*x) if i % 3 == 0 else bq((x[0], M), (x[1], S), (PRICE, F)) if i % 3 == 1 else
                   bq((x[0], S), (x[1], S), (x[2], S), (MV, N), msm=2))
    return out


def same_rows(a, b, rows_a, rows_b, what):
    for i, j in zip(rows_a, rows_b):
        n = int(a.counts[i])
        assert n == b.counts[j] and np.array_equal(a.docs[i, :n], b.docs[j, :n]), f"{what} row {i}"
        assert np.array_equal(a.scores[i, :n].view(np.uint32), b.scores[j, :n].view(np.uint32)), f"{what} row {i}: scores"
        assert a.total_hits[i] == b.total_hits[j] and a.relation[i] == b.relation[j], f"{what} row {i}: totalHits"


def test_flat_queries_inside_a_tree_batch(corpus, batch):
    _, g = corpus
    qs, _ = batch
    s = GpuIndexSearcher(g)
    flats = flat_queries(12)
    mixed = s.search_tree(qs[:6] + flats, RelevanceCollector(100, INT_MAX))
    alone = s.search_batch(flats, RelevanceCollector(100, INT_MAX))
    same_rows(mixed, alone, range(6, 6 + len(flats)), range(len(flats)), "flat in a tree batch")


@pytest.mark.parametrize("threshold", [INT_MAX, 1000])
def test_no_nodes_is_search_bool_ex(corpus, threshold):
    _, g = corpus
    s = GpuIndexSearcher(g)
    flats = flat_queries(24)
    a = s.search_tree(flats, RelevanceCollector(50, threshold))
    b = s.search_batch(flats, RelevanceCollector(50, threshold))
    same_rows(a, b, range(len(flats)), range(len(flats)), f"n_nodes 0, thr={threshold}")
    assert np.array_equal(a.hit_timeout, b.hit_timeout) and np.array_equal(a.terminated_early, b.terminated_early)


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


def _call(g, arrays, k=10):
    carr, ncl, narr, nn, qarr, nq = arrays
    out = [np.zeros(nq * k, np.int32), np.zeros(nq * k, np.float32), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
           np.zeros(nq, np.uint8), np.zeros(nq, np.uint8), np.zeros(nq, np.uint8)]
    return _native.gpu_lib().nrtgpu_search_tree(g.handle, carr, ncl, narr, nn, qarr, nq, k, INT_MAX, 0, None, None,
                                                 *[o.ctypes.data for o in out])


def _arrays(clauses, nodes, queries):
    carr = (_native.Clause * max(len(clauses), 1))(*[_native.Clause(*c) for c in clauses])
    narr = (_native.Node * max(len(nodes), 1))(*[_native.Node(*n) for n in nodes])
    qarr = (_native.Query * len(queries))(*[_native.Query(*q) for q in queries])
    return carr, len(clauses), narr, len(nodes), qarr, len(queries)


@pytest.mark.parametrize("case", range(len(INVALID_TREES)))
def test_invalid_status(corpus, case):
    _, g = corpus
    clauses, nodes, queries, msg = INVALID_TREES[case]
    assert _call(g, _arrays(clauses, nodes, queries)) == 1
    assert msg in _native.gpu_lib().nrtgpu_last_error().decode()


def test_unsupported_status(corpus):
    _, g = corpus
    deep4 = bq((bq((bq((bq((0, S)), M)), M)), M))
    cases = [[bq(*[(bq((t, S)), S) for t in range(9)])], [bq((match(*range(9)), M))],
             [bq((bq(*[(PRICE, S)] * 31), M), (PRICE, S))], [bq((deep4, M))]]
    for qs in cases:
        assert _call(g, compile_tree(qs)) == 3, _native.gpu_lib().nrtgpu_last_error()
    assert _call(g, compile_tree([deep4]), k=1025) == 3
    with pytest.raises(NrtGpuUnsupported):
        GpuIndexSearcher(g).search_tree([deep4], RelevanceCollector(1025, INT_MAX))
    # the flat entry points keep refusing node clauses
    carr, ncl, narr, nn, qarr, nq = compile_tree([bq((match(1, 2), M))])
    out = np.zeros(16, np.int64)
    rc = _native.gpu_lib().nrtgpu_search_bool(g.handle, carr, ncl, qarr, nq, 1, INT_MAX, 0, None, *[out.ctypes.data] * 5)
    assert rc == 1 and "bad clause kind" in _native.gpu_lib().nrtgpu_last_error().decode()
    with pytest.raises(NrtGpuError):
        compile_queries([bq((match(1, 2), M))])
