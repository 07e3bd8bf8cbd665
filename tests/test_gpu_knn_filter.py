"""kNN with a filter query per query vector (KnnQuery.filter, reference KnnUtils.java:135-155), evaluated on the device by
nrtgpu_search_knn_filtered. Every page is compared with the oracle: the filter's match bitmap (oracle.match_bitmap), then
exact brute force over the matching live docs (oracle.knn_exact)."""
import ctypes as C

import numpy as np
import pytest

import oracle
from nrtsearch_b200 import _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, GpuIndex, GpuIndexSearcher, MatchAllDocsQuery, Occur, RangeQuery, TermQuery,
                                   compile_filters)
from test_gpu_knn import assert_certifiable, check

pytestmark = pytest.mark.gpu
GATHER_RATIO = 320   # kKnnGatherRatio: filters matching <= n_vec / 320 docs take the gather path


def filter_shard(n_docs, dims, sim, seed=1, vec_docs=None, doc_base=0, byte_vectors=False):
    """Text field (dense and sparse terms), column 0 single-valued price 0..999, column 1 multi-valued 0..3 values in
    0..99, column 2 = doc id; 10 % of the docs deleted; one vector per doc, or per vec_docs entry."""
    sh = ix.synth_text_shard(n_docs, 2000)
    sh.doc_base = doc_base
    rng = np.random.default_rng(seed)
    cnt = rng.integers(0, 4, n_docs)
    off = np.zeros(n_docs + 1, np.int64)
    np.cumsum(cnt, out=off[1:])
    doc_of = np.repeat(np.arange(n_docs), cnt)
    vals = rng.integers(0, 100, int(off[-1])).astype(np.int64)
    vals = vals[np.lexsort((vals, doc_of))]
    sh.columns = [rng.integers(0, 1000, n_docs).astype(np.int64), vals, np.arange(n_docs, dtype=np.int64)]
    sh.column_has = [None, None, None]
    sh.column_offsets = [None, off, None]
    sh.live_docs = (rng.random(n_docs) >= 0.1).astype(np.uint8)
    n_vec = n_docs if vec_docs is None else len(vec_docs)
    if byte_vectors:
        sh.vectors = rng.integers(-128, 128, size=(n_vec, dims), dtype=np.int8)
    else:
        sh.vectors = ix.synth_vectors(n_vec, dims, seed=ix.SEED_VECTORS + seed)
    sh.vec_similarity = sim
    sh.vec_docs = vec_docs
    return sh


def term_with_df(sh, target):
    return int(np.argmin(np.abs(np.diff(sh.term_off) - target)))


def oracle_filtered(sh, queries, k, filters, boosts=None):
    """The oracle's pages, and per query the eligible docs (filter match & live), by doc."""
    nq = len(queries)
    carr, _, qarr, _, filter_of = compile_filters(filters, nq)
    oix = oracle.OracleIndex(sh)
    live = sh.live_docs.astype(bool)
    vd = np.arange(len(sh.vectors)) if sh.vec_docs is None else sh.vec_docs
    corpus = np.asarray(sh.vectors, np.float32)
    sim = sh.vec_similarity | (0x100 if sh.vectors.dtype == np.int8 else 0)
    wd, ws, wc = np.zeros((nq, k), np.int32), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32)
    eligible = {}
    for f in sorted(set(filter_of.tolist())):
        m = live.copy() if f < 0 else (oracle.match_bitmap(oix, carr, qarr, f).astype(bool) & live)
        eligible[f] = m
        sel = np.nonzero(filter_of == f)[0]
        o, s, c = oracle.knn_exact(corpus, sim, queries[sel], k, filter_docs=m[vd].astype(np.uint8),
                                   boosts=None if boosts is None else boosts[sel])
        wd[sel] = np.where(np.arange(k)[None, :] < c[:, None], vd[np.clip(o, 0, len(vd) - 1)] + sh.doc_base, 0)
        ws[sel], wc[sel] = s, c
    return wd, ws, wc, filter_of, eligible


def run(ctx, sh, queries, k, filters, boosts=None):
    """GPU pages, uncertified count and gather-path count of one filtered call."""
    gix = GpuIndex(ctx, sh)
    try:
        gd, gs, gc = GpuIndexSearcher(gix).knn(queries, k, boosts=boosts, filter_queries=filters)
        lib = _native.gpu_lib()
        unc = lib.nrtgpu_knn_last_uncertified(gix.handle)
        n_gather, ms = C.c_int32(), C.c_float()
        assert lib.nrtgpu_knn_filter_stats(gix.handle, C.byref(n_gather), C.byref(ms)) == 0
    finally:
        gix.close()
    return gd, gs, gc, unc, n_gather.value


def mixed_filters(sh):
    dense, sparse = 0, term_with_df(sh, 200)
    return [
        TermQuery(dense),
        TermQuery(sparse),
        RangeQuery(0, 200, 599),
        RangeQuery(1, 10, 19),                                              # multi-valued: any value in range
        BooleanQuery().add(TermQuery(dense), Occur.MUST).add(RangeQuery(0, 0, 499), Occur.MUST_NOT),
        BooleanQuery(minimum_number_should_match=2).add(TermQuery(1), Occur.SHOULD).add(TermQuery(2), Occur.SHOULD)
        .add(RangeQuery(1, 50, 99), Occur.SHOULD),
        BooleanQuery().add(RangeQuery(0, 0, 799), Occur.FILTER).add(TermQuery(3), Occur.SHOULD),   # SHOULD optional next to a filter
        MatchAllDocsQuery(),
        BooleanQuery(),                                                     # empty BooleanQuery: no hits
        BooleanQuery().add(TermQuery(dense), Occur.MUST_NOT),               # only MUST_NOT: no hits
        None,
    ]


def test_mixed_filter_kinds_in_one_batch(gpu_ctx):
    n, dims, k = 60_000, 64, 20
    sh = filter_shard(n, dims, ix.SIM_L2)
    kinds = mixed_filters(sh)
    nq = 4 * len(kinds)
    queries = ix.synth_vectors(nq, dims, seed=ix.SEED_VQUERIES)
    filters = [kinds[i % len(kinds)] for i in range(nq)]
    gd, gs, gc, _, _ = run(gpu_ctx, sh, queries, k, filters)
    wd, ws, wc, filter_of, _ = oracle_filtered(sh, queries, k, filters)
    assert filter_of.max() == len(kinds) - 2   # equal filters share one index
    check(gd, gs, gc, wd, ws, wc)
    assert (gc[8::len(kinds)] == 0).all() and (gc[9::len(kinds)] == 0).all()


def test_gather_counts_pin_filter_evaluation(gpu_ctx):
    """k >= matches: the count is exactly the number of live matching docs with a vector, for every filter kind."""
    n, dims, k = 120_000, 32, 1024
    sh = filter_shard(n, dims, ix.SIM_COSINE, seed=2)
    sparse = term_with_df(sh, 250)
    kinds = [
        BooleanQuery().add(TermQuery(sparse), Occur.FILTER).add(RangeQuery(0, 0, 699), Occur.FILTER),
        BooleanQuery().add(TermQuery(sparse), Occur.MUST).add(RangeQuery(0, 0, 499), Occur.MUST_NOT),
        BooleanQuery().add(RangeQuery(2, 5_000, 5_300), Occur.FILTER).add(RangeQuery(1, 0, 40), Occur.FILTER),
        BooleanQuery(minimum_number_should_match=2).add(TermQuery(sparse), Occur.SHOULD).add(RangeQuery(2, 0, 299), Occur.SHOULD)
        .add(RangeQuery(0, 0, 499), Occur.SHOULD),
        RangeQuery(2, n - 300, n + 10),
    ]
    queries = ix.synth_vectors(len(kinds), dims, seed=ix.SEED_VQUERIES)
    gd, gs, gc, _, n_gather = run(gpu_ctx, sh, queries, k, kinds)
    wd, ws, wc, filter_of, eligible = oracle_filtered(sh, queries, k, kinds)
    want = np.array([np.count_nonzero(eligible[int(f)]) for f in filter_of])
    assert (want * GATHER_RATIO <= n).all() and (want > 0).all()
    assert n_gather == len(kinds)
    assert np.array_equal(gc, want), (gc, want)
    check(gd, gs, gc, wd, ws, wc)


def test_both_paths_sparse_vec_docs_doc_base(gpu_ctx):
    """300 queries (three 128-row query tiles): filters of <= 64 docs (gather path) and of >= 25 % of the docs (candidate
    GEMM), boosts, a sparse ord -> doc map and doc_base != 0. Certified: the filtered GEMM path alone finds the pages."""
    n_docs, n_vec, dims, k, nq, doc_base = 140_000, 70_000, 32, 20, 300, 1_000_000
    rng = np.random.default_rng(5)
    vec_docs = np.sort(rng.choice(n_docs, n_vec, replace=False)).astype(np.int32)
    sh = filter_shard(n_docs, dims, ix.SIM_COSINE, seed=3, vec_docs=vec_docs, doc_base=doc_base)
    small = [RangeQuery(2, a, a + 63) for a in range(0, 50 * 1000, 1000)]
    large = [RangeQuery(0, 0, 299), BooleanQuery().add(RangeQuery(0, 100, 699), Occur.FILTER).add(TermQuery(0), Occur.MUST)]
    filters = [small[i % len(small)] if i % 3 == 0 else large[i % 2] for i in range(nq)]
    queries = ix.synth_vectors(nq, dims, seed=ix.SEED_VQUERIES)
    boosts = rng.uniform(0.5, 2.0, nq).astype(np.float32)
    wd, ws, wc, filter_of, eligible = oracle_filtered(sh, queries, k, filters, boosts)
    for f in set(filter_of.tolist()):
        if np.count_nonzero(eligible[f]) * GATHER_RATIO > n_vec:
            sel = filter_of == f
            assert_certifiable(sh.vectors, queries[sel], ix.SIM_COSINE, k, eligible=eligible[f][vec_docs])
    gd, gs, gc, unc, n_gather = run(gpu_ctx, sh, queries, k, filters, boosts)
    check(gd, gs, gc, wd, ws, wc)
    assert n_gather == 100, n_gather
    assert unc == 0, unc


@pytest.mark.parametrize("flt", [RangeQuery(0, 0, 499), BooleanQuery().add(RangeQuery(2, 7_000, 7_199), Occur.MUST)])
def test_shared_filter_matches_byte_filter_bit_for_bit(gpu_ctx, flt):
    """One filter index shared by the batch gives the same docs and scores, bit for bit, as nrtgpu_search_knn with that
    filter as bytes: on the candidate GEMM path (50 % filter) and on the gather path (200 docs)."""
    n, dims, k, nq = 80_000, 64, 30, 150
    sh = filter_shard(n, dims, ix.SIM_COSINE, seed=4)
    queries = ix.synth_vectors(nq, dims, seed=ix.SEED_VQUERIES)
    carr, _, qarr, nf, filter_of = compile_filters([flt] * nq, nq)
    assert nf == 1 and (filter_of == 0).all()
    flt_bytes = oracle.match_bitmap(oracle.OracleIndex(sh), carr, qarr, 0)
    gix = GpuIndex(gpu_ctx, sh)
    try:
        s = GpuIndexSearcher(gix)
        a = s.knn(queries, k, filter_queries=[flt] * nq)
        b = s.knn(queries, k, filter_docs=flt_bytes)
    finally:
        gix.close()
    assert np.array_equal(a[2], b[2]) and np.array_equal(a[0], b[0])
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def test_clustered_late_filter_overflow_rerun(gpu_ctx):
    """Filters matching only docs past the 32K warm chunk leave the thresholds at -inf, the first fused chunk overflows
    the survivor buffer, and the unfused rerun must carry the filter rows."""
    n, dims, k = 100_000, 64, 10
    sh = filter_shard(n, dims, ix.SIM_L2, seed=6)
    filters = [RangeQuery(2, 40_000, n), BooleanQuery().add(RangeQuery(2, 50_000, n), Occur.FILTER).add(TermQuery(0), Occur.MUST), None] * 8
    queries = ix.synth_vectors(len(filters), dims, seed=ix.SEED_VQUERIES)
    gd, gs, gc, _, n_gather = run(gpu_ctx, sh, queries, k, filters)
    wd, ws, wc, _, _ = oracle_filtered(sh, queries, k, filters)
    check(gd, gs, gc, wd, ws, wc)
    assert n_gather == 0
    assert (gd[0::3] >= 40_000).all() and (gd[1::3] >= 50_000).all()


def test_simt_stage_dims_100(gpu_ctx):
    n, dims, k = 50_000, 100, 15
    sh = filter_shard(n, dims, ix.SIM_L2, seed=7)
    kinds = mixed_filters(sh) + [RangeQuery(2, 100, 150)]
    queries = ix.synth_vectors(2 * len(kinds), dims, seed=ix.SEED_VQUERIES)
    filters = kinds * 2
    gd, gs, gc, _, n_gather = run(gpu_ctx, sh, queries, k, filters)
    wd, ws, wc, _, _ = oracle_filtered(sh, queries, k, filters)
    check(gd, gs, gc, wd, ws, wc)
    assert n_gather > 0


@pytest.mark.parametrize("sim", [ix.SIM_DOT, ix.SIM_L2])
def test_byte_vectors(gpu_ctx, sim):
    n, dims, k = 40_000, 96, 20
    sh = filter_shard(n, dims, sim, seed=8, byte_vectors=True)
    rng = np.random.default_rng(9)
    kinds = mixed_filters(sh) + [RangeQuery(2, 900, 990)]
    queries = rng.integers(-128, 128, size=(2 * len(kinds), dims)).astype(np.float32)
    filters = kinds * 2
    gd, gs, gc, _, n_gather = run(gpu_ctx, sh, queries, k, filters)
    wd, ws, wc, _, _ = oracle_filtered(sh, queries, k, filters)
    check(gd, gs, gc, wd, ws, wc)
    assert n_gather > 0


def test_invalid_and_unsupported_arguments(gpu_ctx):
    lib = _native.gpu_lib()
    n, dims, k, nq = 5_000, 16, 5, 2
    sh = filter_shard(n, dims, ix.SIM_COSINE, seed=10)
    queries = ix.synth_vectors(nq, dims, seed=ix.SEED_VQUERIES)
    docs, scores, counts = np.zeros((nq, 1100), np.int32), np.zeros((nq, 1100), np.float32), np.zeros(nq, np.int32)

    def call(index, clauses, filters, filter_of, k=k):
        carr = (_native.Clause * max(len(clauses), 1))(*[_native.Clause(*c) for c in clauses])
        qarr = (_native.Query * max(len(filters), 1))(*[_native.Query(*q) for q in filters])
        fo = np.ascontiguousarray(filter_of, np.int32)
        return lib.nrtgpu_search_knn_filtered(index.handle, queries.ctypes.data, nq, k, None, carr, len(clauses), qarr, len(filters),
                                              fo.ctypes.data, None, docs.ctypes.data, scores.ctypes.data, counts.ctypes.data)

    term = (int(Occur.MUST), 0, 5, 1.0, 0, 0)
    ok = ([term], [(0, 1, 0, 0, 0, 0.0)])
    gix = GpuIndex(gpu_ctx, sh)
    try:
        assert call(gix, *ok, [0, -1]) == 0
        assert call(gix, [term], [(0, 1, 0, 1, 3, 1.0)], [0, 0]) == 1                    # has_after on a filter
        assert call(gix, *ok, [1, 0]) == 1 and call(gix, *ok, [0, -2]) == 1               # filter_of out of range
        assert call(gix, [(int(Occur.MUST), 0, 10**6, 1.0, 0, 0)], [(0, 1, 0, 0, 0, 0.0)], [0, 0]) == 1   # term id
        assert call(gix, [(int(Occur.FILTER), 1, 9, 1.0, 0, 5)], [(0, 1, 0, 0, 0, 0.0)], [0, 0]) == 1     # column id
        assert call(gix, *ok, [0, 0], k=0) == 1 and call(gix, *ok, [0, 0], k=1025) == 1
        many = [(int(Occur.SHOULD), 0, t, 1.0, 0, 0) for t in range(9)]                   # 9 term clauses
        assert call(gix, many, [(0, 9, 0, 0, 0, 0.0)], [0, 0]) == 3
        wide = [(int(Occur.FILTER), 1, 0, 1.0, 0, t) for t in range(17)]                  # 17 clauses
        assert call(gix, wide, [(0, 17, 0, 0, 0, 0.0)], [0, 0]) == 3
    finally:
        gix.close()
    sh.vectors = None
    gix = GpuIndex(gpu_ctx, sh)
    try:
        assert call(gix, *ok, [0, 0]) == 1                                                 # no vector field
    finally:
        gix.close()
    with pytest.raises(ValueError):
        GpuIndexSearcher(GpuIndex.__new__(GpuIndex)).knn(queries, k, filter_docs=np.ones(n, np.uint8), filter_queries=[None, None])


def test_filters_past_the_scratch_budget_run_in_groups(gpu_ctx):
    """4M docs make a filter row 500 KB: 300 distinct filters (270 MB of rows against the 128 MB budget) run as two query
    groups, and the 600 distinct term bitmaps of the first group (two terms per filter) are built in several subgroups.
    Odd filters are large (range FILTER minus two terms: candidate GEMM), even ones small (one of two SHOULD terms, msm 1,
    inside a range: gather path); 30 queries have no filter."""
    n, dims, k, n_f = 4_000_000, 16, 10, 300
    rng = np.random.default_rng(12)
    posts = [np.unique(rng.integers(0, n, 2_100)).astype(np.int32) for _ in range(2 * n_f)]
    term_off = np.zeros(len(posts) + 1, np.int64)
    np.cumsum([len(p) for p in posts], out=term_off[1:])
    post_docs = np.concatenate(posts)
    sh = ix.HostShard(n_docs=n, doc_base=0, term_off=term_off, post_docs=post_docs, post_freqs=np.ones(len(post_docs), np.int32),
                      fields=[ix.TextField(None, n, len(post_docs))], columns=[rng.integers(0, 1000, n).astype(np.int64)],
                      column_has=[None], live_docs=(rng.random(n) >= 0.1).astype(np.uint8),
                      vectors=ix.synth_vectors(n, dims, seed=ix.SEED_VECTORS + 12), vec_similarity=ix.SIM_COSINE)
    filters = []
    for i in range(n_f):
        a, b = 2 * i, 2 * i + 1
        if i % 2:
            filters.append(BooleanQuery().add(RangeQuery(0, i, i + 299), Occur.FILTER).add(TermQuery(a), Occur.MUST_NOT)
                           .add(TermQuery(b), Occur.MUST_NOT))
        else:
            filters.append(BooleanQuery(minimum_number_should_match=1).add(TermQuery(a), Occur.SHOULD)
                           .add(TermQuery(b), Occur.SHOULD).add(RangeQuery(0, 0, 599), Occur.FILTER))
    filters += [None] * 30
    queries = ix.synth_vectors(len(filters), dims, seed=ix.SEED_VQUERIES)
    boosts = rng.uniform(0.5, 2.0, len(filters)).astype(np.float32)
    gd, gs, gc, _, n_gather = run(gpu_ctx, sh, queries, k, filters, boosts)
    wd, ws, wc, _, _ = oracle_filtered(sh, queries, k, filters, boosts)
    check(gd, gs, gc, wd, ws, wc)
    assert n_gather == n_f // 2, n_gather
