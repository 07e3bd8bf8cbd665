"""QueryRescorer's second pass (score_docs_kernel: one flat BooleanQuery evaluated on given docs), the whole QueryRescore on
the device (score_docs_kernel + rescore_combine_kernel) and the fetch phase (fetch_columns_kernel), against the oracle
bit for bit. eval_query_on_doc restates the BooleanScorerSupplier rules a third time, beside the probe and window
kernels, so every occur, both score sums and every tf source is covered here:
  - a hand-built 200K-doc shard with doc_base != 0 and deletes;
  - tf-plane terms (df >= n/64) with tf 3..9 and with tf >= 255 (byte 255: exact_freq_slow), non-plane terms with
    tf >= 255, a second text field without norms;
  - an int32 column with missing values, an int64 column, a multi-valued column;
  - hit lists mixing matching, non-matching and deleted docs, duplicates, docs outside the leaf and junk past counts."""
import numpy as np
import pytest

import oracle
import plan_harness as ph
from nrtsearch_b200 import NrtGpuError, NrtGpuUnsupported
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, GpuIndex, GpuIndexSearcher, MatchAllDocsQuery, Occur, RangeQuery,
                                   TermQuery, compile_queries)

pytestmark = pytest.mark.gpu
N = 200_000
DOC_BASE = 3_000_000
C32, C64, CMV = 0, 1, 2
# (field, docs, tf sampler) per term; term ids in this order
PLANE_TF3_9, PLANE_TF255, PLANE_SMALL, BIG_TF, NONPLANE, RARE, F1_PLANE, F1_BIG_TF, COMMON = range(9)
PLANE_TERMS = {PLANE_TF3_9, PLANE_TF255, PLANE_SMALL, F1_PLANE, COMMON}


def make_shard(seed=0x5EC):
    rng = np.random.default_rng(seed)

    def tf(n, lo, hi, big_share=0.0, big=(255, 2000)):
        t = rng.integers(lo, hi + 1, n)
        b = rng.random(n) < big_share
        t[b] = rng.integers(big[0], big[1], int(b.sum()))
        return t

    spec = [(0, N // 16, lambda k: tf(k, 3, 9)),
            (0, N // 40, lambda k: tf(k, 1, 2, 0.1)),
            (0, N // 50, lambda k: tf(k, 1, 4)),
            (0, 600, lambda k: tf(k, 1, 3, 0.5, (255, 700))),
            (0, 2500, lambda k: tf(k, 1, 6)),
            (0, 40, lambda k: tf(k, 1, 2)),
            (1, N // 20, lambda k: tf(k, 1, 3)),
            (1, 2000, lambda k: tf(k, 1, 300, 0.2)),
            (0, N // 2, lambda k: tf(k, 1, 2))]
    lists = []
    for _, df, sampler in spec:
        d = np.sort(rng.choice(N, df, replace=False)).astype(np.int32)
        lists.append((d, sampler(df).astype(np.int32)))
    off = np.zeros(len(lists) + 1, np.int64)
    off[1:] = np.cumsum([len(d) for d, _ in lists])
    term_field = np.array([f for f, _, _ in spec], np.int32)
    lengths = [np.zeros(N, np.int64), np.zeros(N, np.int64)]
    for (f, _, _), (d, t) in zip(spec, lists):
        np.add.at(lengths[f], d, t)
    lengths[0] += rng.integers(1, 40, N)
    byte4 = {int(L): oracle.int_to_byte4(int(L)) for L in np.unique(lengths[0])}
    norms0 = np.array([byte4[int(L)] for L in lengths[0]], np.uint8)
    fields = [ix.TextField(norms0, N, int(lengths[0].sum())),
              ix.TextField(None, int((lengths[1] > 0).sum()), int(lengths[1].sum()))]   # omitNorms
    c32 = rng.integers(-1000, 1000, N).astype(np.int64)
    has32 = (rng.random(N) < 0.8).astype(np.uint8)
    c64 = rng.integers(-2**40, 2**40, N).astype(np.int64)
    nv = rng.integers(0, 4, N)
    offs = np.zeros(N + 1, np.int64)
    np.cumsum(nv, out=offs[1:])
    mv = np.sort(rng.integers(0, 100, (N, 3)), axis=1)
    mvals = np.concatenate([mv[i, :nv[i]] for i in range(N)]).astype(np.int64)
    live = ((np.arange(N) % 13 != 5) & (rng.random(N) >= 0.05)).astype(np.uint8)
    sh = ix.HostShard(n_docs=N, doc_base=DOC_BASE, term_off=off, post_docs=np.concatenate([d for d, _ in lists]),
                      post_freqs=np.concatenate([t for _, t in lists]), fields=fields, term_field=term_field,
                      columns=[c32, c64, mvals], column_has=[has32, None, None], column_offsets=[None, None, offs],
                      live_docs=live)
    return sh


@pytest.fixture(scope="module")
def setup(gpu_ctx):
    sh = make_shard()
    gix = GpuIndex(gpu_ctx, sh)
    yield sh, gix, oracle.OracleIndex(sh)
    gix.close()


def T(t, boost=None):
    return TermQuery(t) if boost is None else BoostQuery(TermQuery(t), boost)


def bq(*clauses, msm=0):
    q = BooleanQuery()
    q.minimum_number_should_match = msm
    for c, o in clauses:
        q.add(c, o)
    return q


S, M, F, NOT = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
QUERIES = [
    bq((T(PLANE_TF3_9), S), (T(PLANE_TF255), S)),
    bq((T(PLANE_TF3_9), M), (T(BIG_TF), S)),                                   # ReqOptSumScorer: float add
    bq((T(COMMON), M), (T(PLANE_TF255), S), (T(BIG_TF), S), msm=1),            # msm > 0: double add
    bq((T(PLANE_SMALL), M), (RangeQuery(C32, -500, 500), F), (T(NONPLANE), NOT)),
    bq((T(F1_PLANE), S), (T(F1_BIG_TF), S), (T(BIG_TF), S)),                   # the field without norms
    BoostQuery(bq((T(PLANE_TF3_9), S), (T(F1_PLANE, 3.0), S)), 0.75),
    MatchAllDocsQuery(),
    bq(*[(T(t), S) for t in (PLANE_TF3_9, PLANE_TF255, PLANE_SMALL, BIG_TF, NONPLANE, RARE)], msm=2),   # 6 term clauses
    bq((T(COMMON), M), *[(T(t), S) for t in (PLANE_TF3_9, PLANE_TF255, PLANE_SMALL, BIG_TF, NONPLANE, F1_PLANE)],
       (T(RARE), NOT)),                                                        # 8 term clauses
    bq((RangeQuery(CMV, 10, 20), F), (T(PLANE_TF255), S)),                     # range on the multi-valued column
    bq((BoostQuery(RangeQuery(C64, 0, 2**40), 2.0), M), (T(F1_BIG_TF), S)),
    BooleanQuery(),                                                            # no clauses: matches nothing
    bq((T(PLANE_TF3_9), S), msm=2),                                            # msm > #SHOULD: matches nothing
    T(RARE),
    bq((T(COMMON), NOT)),                                                      # MUST_NOT only: matches nothing
    bq((T(PLANE_SMALL), M), (BoostQuery(MatchAllDocsQuery(), 0.5), S), (T(F1_BIG_TF), S)),
]


def test_shard_has_the_tf_sources_it_claims(setup):
    sh, _, _ = setup
    plane, _ = ph.index_rules(N, sh.term_off)
    assert {t for t in range(sh.n_terms) if plane[t] >= 0} == PLANE_TERMS
    tf = [sh.post_freqs[sh.term_off[t]:sh.term_off[t + 1]] for t in range(sh.n_terms)]
    assert tf[PLANE_TF3_9].min() == 3 and tf[PLANE_TF3_9].max() == 9
    assert (tf[PLANE_TF255] >= 255).any() and (tf[BIG_TF] >= 255).any() and (tf[F1_BIG_TF] >= 255).any()


def hit_lists(sh, oix, n_hits, seed):
    """per query: matching, non-matching and deleted docs, duplicates and docs outside the leaf (global ids), in random
    order; counts below n_hits, with junk after them"""
    rng = np.random.default_rng(seed)
    carr, _, qarr, nq = compile_queries(QUERIES)
    dead = np.nonzero(sh.live_docs == 0)[0]
    outside = np.array([DOC_BASE - 1, 0, -7, DOC_BASE + N, DOC_BASE + N + 1000, 2**31 - 1, -2**31], np.int64)
    docs = np.zeros((nq, n_hits), np.int32)
    counts = np.zeros(nq, np.int32)
    for q in range(nq):
        m = np.nonzero(oracle.match_bitmap(oix, carr, qarr, q))[0]
        parts = [rng.choice(m, min(len(m), n_hits // 3), replace=False) if len(m) else np.zeros(0, np.int64),
                 rng.integers(0, N, n_hits // 4), rng.choice(dead, n_hits // 16)]
        local = np.concatenate(parts)
        local = np.concatenate([local, rng.choice(local, n_hits // 16)])   # duplicates
        glob = np.concatenate([local + DOC_BASE, outside])
        glob = glob[rng.permutation(len(glob))][:n_hits]
        counts[q] = len(glob) - int(rng.integers(0, 20))
        docs[q, :len(glob)] = glob
        docs[q, counts[q]:] = rng.integers(-2**31, 2**31 - 1, n_hits - counts[q])   # junk past counts
    return docs, counts


@pytest.mark.parametrize("with_counts", [True, False])
def test_score_docs_matches_oracle(setup, with_counts):
    sh, gix, oix = setup
    docs, counts = hit_lists(sh, oix, 3000, 11)
    cn = counts if with_counts else None
    m, s = GpuIndexSearcher(gix).score_docs(QUERIES, docs, cn)
    carr, _, qarr, nq = compile_queries(QUERIES)
    wm, ws = oracle.score_docs(oix, carr, qarr, nq, docs, cn)
    for q in range(nq):
        assert np.array_equal(m[q], wm[q]), f"query {q}: matches differ at {np.nonzero(m[q] != wm[q])[0][:5]}"
        assert np.array_equal(s[q].view(np.uint32), ws[q].view(np.uint32)), f"query {q}: scores differ"
    matched = wm.sum(axis=1)
    assert (matched[[0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 13, 15]] > 0).all() and not matched[[11, 12, 14]].any()
    if with_counts:
        assert not any(m[q, counts[q]:].any() for q in range(nq))


WEIGHTS = [(1.0, 1.0), (0.5, 2.5), (1.0, 0.0), (0.0, 1.0)]


@pytest.mark.parametrize("weights", WEIGHTS)
def test_rescore_query_matches_oracle(setup, weights):
    sh, gix, oix = setup
    n_hits = 4096
    docs, counts = hit_lists(sh, oix, n_hits, 12)
    docs &= np.int32(0x7fffffff)   # first-pass hits are doc ids >= 0 (ties are broken by doc id)
    nq = len(QUERIES)
    counts[:4] = [0, 1, n_hits, n_hits - 1]
    rng = np.random.default_rng(13)
    first = np.round(rng.random((nq, n_hits)) * 8, 1).astype(np.float32)   # few distinct scores: ties by doc id
    carr, _, qarr, _ = compile_queries(QUERIES)
    wm, ws = oracle.score_docs(oix, carr, qarr, nq, docs, counts)
    s = GpuIndexSearcher(gix)
    for window in (1, 40, n_hits + 1):
        d, r, c = s.rescore_query(QUERIES, docs, first, counts, window, *weights)
        for q in range(nq):
            n = int(counts[q])
            od, os_ = oracle.rescore_combine(docs[q, :n], first[q, :n], wm[q, :n], ws[q, :n], *weights)
            keep = min(n, window)
            assert c[q] == keep, f"window {window} query {q}: count"
            assert np.array_equal(d[q, :keep], od[:keep]), f"window {window} query {q}: docs differ"
            assert np.array_equal(r[q, :keep].view(np.uint32), os_[:keep].view(np.uint32)), f"window {window} query {q}: scores"


def test_rescore_query_refusals(setup):
    _, gix, _ = setup
    s = GpuIndexSearcher(gix)
    qs = QUERIES[:2]
    docs, scores = np.full((2, 4097), DOC_BASE, np.int32), np.ones((2, 4097), np.float32)
    with pytest.raises(NrtGpuUnsupported, match="more than 4096 hits per query"):
        s.rescore_query(qs, docs, scores, np.array([1, 1], np.int32), 10, 1.0, 1.0)
    for bad in (-1, 4097):
        with pytest.raises(NrtGpuError, match="counts out of range") as e:
            s.rescore_query(qs, docs[:, :4096], scores[:, :4096], np.array([5, bad], np.int32), 10, 1.0, 1.0)
        assert e.value.status == 1


def test_fetch_columns_matches_host(setup):
    sh, gix, _ = setup
    rng = np.random.default_rng(14)
    local = rng.integers(-3000, N + 3000, 70_000)                 # some outside the leaf: has 0, value 0
    glob = (local + DOC_BASE).astype(np.int32)
    vals, has = GpuIndexSearcher(gix).fetch_columns([C64, C32, C32], glob)
    inside = (local >= 0) & (local < N)
    li = np.clip(local, 0, N - 1)
    want_has32 = inside & (sh.column_has[C32][li] != 0)
    assert np.array_equal(has[0], inside.astype(np.uint8)) and np.array_equal(has[1], want_has32.astype(np.uint8))
    assert np.array_equal(vals[0], np.where(inside, sh.columns[C64][li], 0))          # int64 storage
    assert np.array_equal(vals[1], np.where(want_has32, sh.columns[C32][li], 0))      # int32 storage, missing -> 0
    assert np.array_equal(vals[2], vals[1]) and np.array_equal(has[2], has[1])
    assert (np.abs(sh.columns[C64]) > 2**31).any() and (sh.columns[C32] < 0).any()
    with pytest.raises(NrtGpuUnsupported, match="multi-valued column"):
        GpuIndexSearcher(gix).fetch_columns([CMV], glob[:10])
