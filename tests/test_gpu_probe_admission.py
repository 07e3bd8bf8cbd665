"""posting_probe_kernel, pure disjunctions: a candidate is scored a warp at a time and only a key above the query's
threshold enters the CTA's 1024-entry buffer. This corpus sends far more than 1024 admitted keys through one work item
(top_k 512, a few distinct norms and small tfs: thousands of docs share a score and are ordered by doc id alone), with
saturated 2-bit plane codes (tf >= 3, the exact byte comes from the byte plane) and tf >= 255 (the exact frequency
comes from the postings), in both score modes and on a searchAfter page. Oracle = exhaustive CPU evaluation."""
import numpy as np
import pytest

import oracle
from helpers import assert_same_hits
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, GpuIndex, GpuIndexSearcher, Occur, RelevanceCollector, ScoreDoc,
                                   TermQuery, compile_queries)

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
N_DOCS = 300_000
TOP_K = 512


def _postings(rng, docs, p_sat, p_huge):
    """tf 1 or 2 for most docs, 3..9 (a saturated plane code) for a share p_sat, 255..400 for a share p_huge"""
    tf = rng.integers(1, 3, size=len(docs))
    u = rng.random(len(docs))
    tf[u < p_sat] = rng.integers(3, 10, size=int((u < p_sat).sum()))
    tf[u < p_huge] = rng.integers(255, 401, size=int((u < p_huge).sum()))
    return docs.astype(np.int32), tf.astype(np.int32)


@pytest.fixture(scope="module")
def corpus():
    rng = np.random.default_rng(31)
    lists = [
        _postings(rng, np.arange(N_DOCS), 0.05, 0.002),                                   # every doc (tf plane)
        _postings(rng, np.arange(0, N_DOCS, 2), 0.10, 0.001),                             # every second doc (tf plane)
        _postings(rng, np.arange(0, N_DOCS, 7), 0.02, 0.0),                               # every 7th doc (tf plane)
        _postings(rng, np.sort(rng.choice(N_DOCS, 3_000, replace=False)), 0.3, 0.01),     # no plane: searched
        _postings(rng, np.sort(rng.choice(N_DOCS, 40, replace=False)), 0.0, 0.0),         # rare
    ]
    term_off = np.zeros(len(lists) + 1, dtype=np.int64)
    term_off[1:] = np.cumsum([len(d) for d, _ in lists])
    post_docs = np.concatenate([d for d, _ in lists])
    post_freqs = np.concatenate([f for _, f in lists])
    norms = rng.choice(np.array([12, 20, 28], dtype=np.uint8), size=N_DOCS)   # three field lengths: many equal scores
    sh = ix.HostShard(n_docs=N_DOCS, doc_base=0, term_off=term_off, post_docs=post_docs, post_freqs=post_freqs,
                      fields=[ix.TextField(norms, N_DOCS, int(post_freqs.sum()))])
    sh.term_df = np.diff(term_off).astype(np.int64)
    return sh


def disj(terms):
    q = BooleanQuery()
    for t in terms:
        q.add(TermQuery(int(t)), Occur.SHOULD)
    return q


QUERIES = [[0], [0, 1], [1, 0], [0, 1, 2], [1, 2, 3], [0, 1, 2, 3], [2, 3], [1, 3], [3, 4], [0, 4], [2, 1, 4, 0]]


def run(gpu_ctx, sh, qs, threshold, search_after=None):
    gix = GpuIndex(gpu_ctx, sh)
    try:
        res = GpuIndexSearcher(gix).search_batch(qs, RelevanceCollector(TOP_K, threshold), search_after=search_after)
    finally:
        gix.close()
    carr, ncl, qarr, nq = compile_queries(qs, search_after)
    want = oracle.search_compiled(oracle.OracleIndex(sh), carr, ncl, qarr, nq, TOP_K)
    return (res.docs, res.scores, res.counts, res.total_hits, res.relation), want


@pytest.mark.parametrize("threshold", [INT_MAX, 1000])
def test_admission_overflow_pages(gpu_ctx, corpus, threshold):
    qs = [disj(t) for t in QUERIES]
    got, want = run(gpu_ctx, corpus, qs, threshold)
    assert_same_hits(got, want, what=f"page 1 thr={threshold}")
    if threshold == INT_MAX:
        assert (got[4] == 0).all(), "ScoreMode.COMPLETE must report exact counts"
    full = [q for q in range(len(qs)) if got[2][q] == TOP_K]
    assert len(full) >= len(qs) - 2
    # the next page starts inside a run of equal scores: the after key separates docs by id alone
    after = [ScoreDoc(int(got[0][q, TOP_K - 1]), float(got[1][q, TOP_K - 1])) for q in full]
    page2, want2 = run(gpu_ctx, corpus, [qs[q] for q in full], threshold, search_after=after)
    assert_same_hits(page2, want2, check_total=threshold == INT_MAX, what=f"page 2 thr={threshold}")
