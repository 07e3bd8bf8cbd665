"""The second-pass reference of tree and phrase rescore queries (tests/rescore_tree_reference.py) on the CPU: QueryTest's
rescore by a sloppy phrase on its addDocs.txt corpus, hand-derived trees where a node's float rounding differs from the
flat clause list's, and the hit-list rules (entries past the count, docs outside the shard, deleted docs)."""
import numpy as np
import pytest

import phrase_reference as pr
import rescore_tree_reference as rr
from helpers import shard_from_token_docs
from nrtsearch_b200.search import BooleanQuery, BoostQuery, DisjunctionMaxQuery, Occur, PhraseQuery, RangeQuery, TermQuery

S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
FIRST, VENDOR, AGAIN, SECOND = 0, 1, 2, 3
E = float(2.0 ** -24)   # half an ulp of 1.0f


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(TermQuery(int(c)) if isinstance(c, (int, np.integer)) else c, o)
    return q


@pytest.fixture(scope="module")
def vendors(built):
    """addDocs.txt's vendor_name (doc_id 1, 2 = shard docs 0, 1), position increment gap 100"""
    docs = [[[[FIRST, VENDOR], [FIRST, AGAIN]]], [[[SECOND, VENDOR], [SECOND, AGAIN]]]]
    return pr.shard_from_tokens(docs, [0, 0, 0, 0], 1)


def test_query_test_rescore_by_a_sloppy_phrase(vendors):
    # first pass: "vendor" (both docs, equal scores: doc 0 first); rescore by "second again"~1 at (1.0, 4.0), window 2
    d, s, c, _, _ = pr.search(vendors, [TermQuery(VENDOR)], 10)
    assert list(d[0, :c[0]]) == [0, 1] and s[0, 0] == s[0, 1]
    first = s[0, 0]
    m, s2 = rr.score_docs(vendors, [PhraseQuery([SECOND, AGAIN], slop=1)], d[:, :2], c)
    assert list(m[0]) == [0, 1] and s2[0, 1] == np.float32(0.3979403)
    rd, rs, rc = rr.rescore(d[:, :2], s[:, :2], m, s2, c, 2, 1.0, 4.0)
    assert rc[0] == 2 and list(rd[0]) == [1, 0]
    assert rs[0, 0] == np.float32(1.0 * float(first) + 4.0 * float(np.float32(0.3979403)))
    assert rs[0, 1] == np.float32(1.0 * float(first))
    # window 1 keeps doc_id 2 alone, as QueryTest's page of one hit
    assert rr.rescore(d[:, :2], s[:, :2], m, s2, c, 1, 1.0, 4.0)[2][0] == 1


@pytest.fixture(scope="module")
def tiny(built):
    sh, _ = shard_from_token_docs([[["a"], ["a", "b"], ["b"], ["c"]]], columns=[np.array([1, 2, 3, 4], np.int64)])
    sh.doc_base = 100
    return sh


def const(c, lo=1, hi=4):
    """a constant-score leaf scoring c on the docs whose column value is in [lo, hi]"""
    return BoostQuery(RangeQuery(0, lo, hi), c)


HITS = np.array([[103, 101, 100, 102]], np.int32)
FIRST_SCORES = np.array([[4.0, 3.0, 2.0, 1.0]], np.float32)


def test_two_level_bool_rounds_at_each_node(tiny):
    # (float)(1 + 2^-24) = 1.0 at the inner node, + 2^-24 at the root rounds to 1.0 again; the flat list is 1 + 2^-23
    nested = bq((bq((const(1.0), M), (const(E), M)), M), (bq((const(E), M)), M))
    flat = bq((const(1.0), M), (const(E), M), (const(E), M))
    m, s = rr.score_docs(tiny, [nested, flat], np.repeat(HITS, 2, 0))
    assert m.all() and (s[0] == np.float32(1.0)).all() and (s[1] == np.float32(1.0 + 2 * E)).all()
    # rescore (0, 1): all tie at 1.0 and sort by doc; the flat query's second pass gives the same order
    d, sc, c = rr.rescore(np.repeat(HITS, 2, 0), np.repeat(FIRST_SCORES, 2, 0), m, s, [4, 4], 3, 0.0, 1.0)
    assert list(c) == [3, 3] and list(d[0, :3]) == [100, 101, 102] and (sc[0, :3] == 1.0).all()
    # (1, 1): the first-pass order survives, each score shifted by the node's float
    d, sc, _ = rr.rescore(HITS, FIRST_SCORES, m[:1], s[:1], [4], 4, 1.0, 1.0)
    assert list(d[0]) == [103, 101, 100, 102] and list(sc[0]) == [5.0, 4.0, 3.0, 2.0]


def test_dismax_rescore(tiny):
    # DisjunctionMaxQuery([0.5 on all, 1.0 on docs 1..3, 0.25 on docs 2..3], 0.5): 0.5, 1.25, 1.375, 1.375
    dm = DisjunctionMaxQuery([const(0.5), const(1.0, 2, 4), const(0.25, 3, 4)], 0.5)
    m, s = rr.score_docs(tiny, [dm], HITS)
    assert list(m[0]) == [1, 1, 1, 1] and list(s[0]) == [1.375, 1.25, 0.5, 1.375]
    d, sc, c = rr.rescore(HITS, FIRST_SCORES, m, s, [4], 40, 1.0, 4.0)
    # 103: 4 + 4 * 1.375, 101: 3 + 4 * 1.25, 102: 1 + 4 * 1.375, 100: 2 + 4 * 0.5
    assert c[0] == 4 and list(d[0]) == [103, 101, 102, 100] and list(sc[0]) == [9.5, 8.0, 6.5, 4.0]
    # at tie_breaker 0 the flat sum of the matching disjuncts would be 1.75 / 1.5; the node keeps the max alone
    m0, s0 = rr.score_docs(tiny, [DisjunctionMaxQuery([const(0.5), const(1.0, 2, 4), const(0.25, 3, 4)], 0.0)], HITS)
    assert list(s0[0]) == [1.0, 1.0, 0.5, 1.0]


def test_hit_list_rules(tiny):
    tiny.live_docs = np.array([1, 1, 0, 1], np.uint8)
    try:
        q = bq((const(1.0), S))
        docs = np.array([[99, 100, 102, 104, 103, 101], [101, 101, 103, 100, 0, 0]], np.int32)
        m, s = rr.score_docs(tiny, [q, q], docs, counts=[6, 3])
        # below doc_base, deleted, at doc_base + n_docs: 0; past the count: 0; duplicates are scored each time
        assert m.tolist() == [[0, 1, 0, 0, 1, 1], [1, 1, 1, 0, 0, 0]]
        assert (s[m == 0] == 0).all() and (s[m == 1] == 1.0).all()
    finally:
        tiny.live_docs = None
