"""The query-tree reference (tests/tree_reference.py) on the CPU: it equals the oracle bit for bit on flat queries, and
hand-derived constant-score trees pin its rounding rules -- where a nested node's float differs from the flat clause list's
double sum, at two and three levels, DisjunctionMaxQuery at tie_breaker 0 and 0.5, and nodes that match nothing."""
import numpy as np
import pytest

import oracle
import tree_reference as tr
from helpers import assert_same_hits, shard_from_token_docs
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, MatchAllDocsQuery, Occur, RangeQuery, ScoreDoc,
                                   TermQuery, compile_queries)

S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
E = float(2.0 ** -24)   # half an ulp of 1.0f


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(TermQuery(int(c)) if isinstance(c, (int, np.integer)) else c, o)
    return q


# ---------------------------------------------------------------- flat queries: the oracle, bit for bit

@pytest.fixture(scope="module")
def synth(built):
    sh = ix.synth_text_shard(30_000, 3_000, min_len=4, poisson_mean=10.0)
    sh.columns = [ix.synth_int_column(sh.n_docs)]
    sh.column_has = [None]
    rng = np.random.default_rng(5)
    sh.live_docs = (rng.random(sh.n_docs) > 0.1).astype(np.uint8)
    return sh


def test_flat_trees_equal_the_oracle(synth):
    terms = ix.synth_query_terms(48, 5, 3_000, log10_lo=0.3, log10_hi=3.0)
    r = RangeQuery(0, 100_000, 700_000)
    qs = []
    for i, t in enumerate(terms):
        k = i % 6
        if k == 0:
            qs.append(bq(*[(x, S) for x in t[:3]]))
        elif k == 1:
            qs.append(bq((t[0], M), (t[1], S), (t[2], S), (r, F)))
        elif k == 2:
            qs.append(bq((t[0], S), (t[1], S), (t[2], S), (t[3], N), msm=2))
        elif k == 3:
            qs.append(BoostQuery(bq((BoostQuery(TermQuery(int(t[0])), 2.5), S), (BoostQuery(r, 0.7), S)), 1.3))
        elif k == 4:
            qs.append(bq((MatchAllDocsQuery(), M), (t[0], S), (t[1], N)))
        else:
            qs.append(bq((t[0], F), (t[1], M), (r, M)))
    oix = oracle.OracleIndex(synth)
    for k in (1, 10, 100):
        carr, ncl, qarr, nq = compile_queries(qs)
        want = oracle.search_compiled(oix, carr, ncl, qarr, nq, k)
        got = tr.search(synth, qs, k, oix=oix)
        assert_same_hits(got, want, what=f"k={k}")
        assert np.array_equal(got[3], want[3])
    # searchAfter: the oracle's second page
    first = tr.search(synth, qs, 10, oix=oix)
    after = [ScoreDoc(int(first[0][q, 9]), float(first[1][q, 9])) if first[2][q] == 10 else None for q in range(len(qs))]
    carr, ncl, qarr, nq = compile_queries(qs, after)
    assert_same_hits(tr.search(synth, qs, 10, after, oix=oix), oracle.search_compiled(oix, carr, ncl, qarr, nq, 10))


# ---------------------------------------------------------------- hand-derived constant-score trees

@pytest.fixture(scope="module")
def tiny(built):
    sh, vocab = shard_from_token_docs([[["a"], ["a", "b"], ["b"], ["c"]]], columns=[np.array([1, 2, 3, 4], np.int64)])
    return sh


def const(c, lo=1, hi=4):
    """a constant-score leaf scoring c on the docs whose column value is in [lo, hi]"""
    return BoostQuery(RangeQuery(0, lo, hi), c)


def scores_of(sh, q):
    """{doc: score} of every match"""
    d, s, c, t, _ = tr.search(sh, [q], 4)
    assert t[0] == c[0]
    return {int(d[0, i]): float(s[0, i]) for i in range(c[0])}


def test_double_sums_inside_a_node(tiny):
    # MUST sum in double: 1 + 2^-24 + 2^-24 = 1 + 2^-23 exactly (a chain of float adds would stay at 1.0)
    q = bq((bq((const(1.0), M), (const(E), M), (const(E), M)), M))
    assert scores_of(tiny, q) == {d: 1.0 + 2 * E for d in range(4)}
    # flat, the same three clauses at the root
    assert scores_of(tiny, bq((const(1.0), M), (const(E), M), (const(E), M))) == {d: 1.0 + 2 * E for d in range(4)}


def test_nesting_rounds_at_every_node_two_levels(tiny):
    # (float)(1 + 2^-24) = 1.0 (a tie, to even); the root adds 2^-24 to a float 1.0 and rounds to 1.0 again
    q = bq((bq((const(1.0), M), (const(E), M)), M), (bq((const(E), M)), M))
    assert scores_of(tiny, q) == {d: 1.0 for d in range(4)}
    # the same in SHOULD sums
    q = bq((bq((const(1.0), S), (const(E), S)), S), (const(E), S))
    assert scores_of(tiny, q) == {d: 1.0 for d in range(4)}
    assert scores_of(tiny, bq((const(1.0), S), (const(E), S), (const(E), S))) == {d: 1.0 + 2 * E for d in range(4)}


def test_nesting_three_levels_and_req_opt(tiny):
    inner = bq((bq((const(E), S), (const(E), S)), M))                   # (float)(2^-24 + 2^-24) = 2^-23
    q = bq((const(1.0), M), (bq((inner, S)), S))                         # ReqOptSumScorer: 1.0f + 2^-23f (float add)
    assert scores_of(tiny, q) == {d: 1.0 + 2 * E for d in range(4)}
    q = bq((const(1.0), M), (bq((inner, S)), S), msm=1)                  # msm > 0: the double add, the same value here
    assert scores_of(tiny, q) == {d: 1.0 + 2 * E for d in range(4)}
    # only docs 1..3 have the optional part: doc 0 scores the required float alone
    q = bq((const(1.0), M), (bq((const(0.5, 2, 4), S), (const(0.25, 2, 4), S)), S))
    assert scores_of(tiny, q) == {0: 1.0, 1: 1.75, 2: 1.75, 3: 1.75}


@pytest.mark.parametrize("tie,want", [(0.0, {0: 0.5, 1: 1.0, 2: 1.0, 3: 1.0}), (0.5, {0: 0.5, 1: 1.25, 2: 1.375, 3: 1.375})])
def test_dismax(tiny, tie, want):
    dm = DisjunctionMaxQuery([const(0.5), const(1.0, 2, 4), const(0.25, 3, 4)], tie)
    assert scores_of(tiny, dm) == want
    assert scores_of(tiny, bq((dm, M), (const(0.0, 4, 4), N))) == {d: want[d] for d in range(3)}


def test_dismax_max_moves_into_the_sum(tiny):
    # streamed in clause order: 1.0 then 2^-24 (others = 2^-24), or 2^-24 then 1.0 (the old max 2^-24 moves into others):
    # either way (float)(1 + 2^-24 * 1) = 1.0, and with three: (float)(1 + 2 * 2^-24) = 1 + 2^-23
    for order in ([const(1.0), const(E)], [const(E), const(1.0)]):
        assert scores_of(tiny, DisjunctionMaxQuery(order, 1.0)) == {d: 1.0 for d in range(4)}
    assert scores_of(tiny, DisjunctionMaxQuery([const(E), const(1.0), const(E)], 1.0)) == {d: 1.0 + 2 * E for d in range(4)}


def test_nodes_that_match_nothing(tiny):
    empty_msm = bq((const(1.0), S), (const(2.0), S), msm=3)
    all_not = bq((const(1.0, 1, 1), N), (const(1.0, 2, 2), N))
    no_clause = BooleanQuery()
    assert scores_of(tiny, bq((empty_msm, M), (const(1.0), S))) == {}
    assert scores_of(tiny, bq((empty_msm, S), (const(1.0, 2, 3), S))) == {1: 1.0, 2: 1.0}
    assert scores_of(tiny, bq((all_not, F), (const(1.0), S))) == {}
    assert scores_of(tiny, bq((all_not, S), (const(0.5), S))) == {d: 0.5 for d in range(4)}
    assert scores_of(tiny, bq((no_clause, S), (const(0.5, 4, 4), S))) == {3: 0.5}
    assert scores_of(tiny, bq((DisjunctionMaxQuery([], 0.0), M))) == {}
    # excluded by a subtree: MUST_NOT (a | b) removes docs 0..2
    assert scores_of(tiny, bq((MatchAllDocsQuery(), M), (bq((TermQuery(0), S), (TermQuery(1), S)), N))) == {3: 1.0}
