"""ConstantScoreQuery and MinScoreQuery in the references (tests/score_nodes_reference.py), on the CPU: the object-level
reference pinned to the known answers of the reference project's ConstantScoreQueryTest and MinThresholdQueryTest and to
hand-computed floats at the edges, the array-level one over compile_tree held to the same answers, then the two compared
over generated trees holding both (tests/score_nodes_gen.py), so the Python compiler's node boosts, restarted folds and
MinScoreQuery(q, 0) unwrapping are under test."""
import math

import numpy as np
import pytest

import oracle
import query_gen as qg
import score_nodes_gen as sg
import score_nodes_reference as snr
from helpers import shard_from_token_docs
from nrtsearch_b200.search import (BooleanClause, BooleanQuery, BoostQuery, ConstantScoreQuery, DisjunctionMaxQuery,
                                   MinScoreQuery, Occur, TermQuery, compile_tree)
from test_query_reference import same_pages, shadow, small_shard, with_shadow_columns

S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
F32 = np.float32


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(c, o)
    return q


def page(sh, q, k=10):
    d, s, c, t = snr.ScoreNodeReference(sh).search([q], k)
    return d[0, :c[0]].tolist(), s[0, :c[0]], int(t[0])


def compiled_page(sh, q, k=10):
    d, s, c, t, _ = snr.search(sh, [q], k)
    return d[0, :c[0]].tolist(), s[0, :c[0]], int(t[0])


# ---------------------------------------------------------------- known answers

CONSTANT_DOCS = ["t1 t2 t3", "t1 t3", "t4 t5 t6", "t2 t6 t7", "t1 t2 t8"]   # ConstantScoreQueryTest
MIN_DOCS = ["test document one", "test test document two", "test test test document three"]   # MinThresholdQueryTest


@pytest.fixture(scope="module")
def constant_shard(built):
    return shard_from_token_docs([[d.split() for d in CONSTANT_DOCS]])


@pytest.fixture(scope="module")
def min_shard(built):
    return shard_from_token_docs([[d.split() for d in MIN_DOCS]])


def test_constant_score_known_answers(constant_shard):
    sh, v = constant_shard
    t2 = TermQuery(v[(0, "t2")])
    for fn in (page, compiled_page):
        d, s, t = fn(sh, ConstantScoreQuery(t2))
        assert d == [0, 3, 4] and t == 3 and s.tolist() == [1.0, 1.0, 1.0]
        d, s, t = fn(sh, BoostQuery(ConstantScoreQuery(t2), 5.0))
        assert d == [0, 3, 4] and s.tolist() == [5.0, 5.0, 5.0]
        # boosts inside are ignored; boosts above two wrappers multiply outermost first
        d, s, t = fn(sh, BoostQuery(ConstantScoreQuery(BoostQuery(t2, 7.0)), 5.0))
        assert s.tolist() == [5.0] * 3
        d, s, t = fn(sh, bq((ConstantScoreQuery(t2), S), (TermQuery(v[(0, "t1")]), S)))
        assert d == [0, 4, 3, 1] and t == 4 and s[2] == 1.0 and s[3] < 1.0 < s[0]


def test_min_threshold_known_answers(min_shard):
    sh, v = min_shard
    test = TermQuery(v[(0, "test")])
    d0, s0, t0 = page(sh, test)
    assert t0 == 3 and (s0 > 0).all()
    for fn in (page, compiled_page):
        d, s, t = fn(sh, MinScoreQuery(test, 0.5))
        assert set(d) <= set(d0) and (s >= F32(0.5)).all() and t == len(d)
        d, s, t = fn(sh, MinScoreQuery(test, 0.0))   # threshold 0: every hit, as the query itself
        assert d == d0 and np.array_equal(s.view(np.uint32), s0.view(np.uint32)) and t == t0


def test_min_score_edges_against_hand_computed_floats(min_shard):
    sh, v = min_shard
    test, doc = TermQuery(v[(0, "test")]), TermQuery(v[(0, "document")])
    d0, s0, _ = page(sh, test)
    sd = dict(zip(d0, s0))
    _, sdoc, _ = page(sh, doc)
    sdoc = dict(zip(page(sh, doc)[0], sdoc))
    mid = F32(sd[1])                       # doc 1's exact score: the boundary
    above = {x for x in d0 if sd[x] >= mid}
    assert 0 < len(above) < 3
    for fn in (page, compiled_page):
        d, s, _ = fn(sh, MinScoreQuery(test, float(mid)))
        assert set(d) == above and 1 in d                          # a doc whose score equals the threshold passes
        d, _, _ = fn(sh, MinScoreQuery(test, float(np.nextafter(mid, F32(np.inf)))))
        assert 1 not in d and set(d) == {x for x in d0 if sd[x] > mid}
        assert fn(sh, MinScoreQuery(test, math.nan))[2] == 0       # NaN: nothing
        # under FILTER the wrapped query still scores for its test; the FILTER adds nothing to the score
        d, s, _ = fn(sh, bq((doc, M), (MinScoreQuery(test, float(mid)), F)))
        assert set(d) == above and all(s[i] == sdoc[x] for i, x in enumerate(d))
        # under MUST_NOT: the docs below the threshold
        d, _, _ = fn(sh, bq((doc, M), (MinScoreQuery(test, float(mid)), N)))
        assert set(d) == set(d0) - above
        # under CONSTANT: filters by score, scores the constant
        d, s, _ = fn(sh, BoostQuery(ConstantScoreQuery(MinScoreQuery(test, float(mid))), 3.0))
        assert set(d) == above and s.tolist() == [3.0] * len(above)
        # a boost above multiplies after the test (the set is that of the unboosted threshold)
        d, s, _ = fn(sh, BoostQuery(MinScoreQuery(test, float(mid)), 2.5))
        assert set(d) == above and all(s[i] == F32(sd[x] * F32(2.5)) for i, x in enumerate(d))
        # a boost inside is part of the tested score
        d, s, _ = fn(sh, MinScoreQuery(BoostQuery(test, 2.0), float(F32(mid * F32(2.0)))))
        assert set(d) == above and all(s[i] == F32(sd[x] * F32(2.0)) for i, x in enumerate(d))
        # a boost above a threshold of 0 folds into the query (QueryNodeMapper unwraps it)
        d, s, _ = fn(sh, BoostQuery(MinScoreQuery(BoostQuery(test, 0.1), 0.0), 1.75))
        want = page(sh, BoostQuery(BoostQuery(test, 0.1), 1.75))
        assert d == want[0] and np.array_equal(s.view(np.uint32), want[1].view(np.uint32))


def test_negative_threshold_is_refused(min_shard):
    sh, v = min_shard
    with pytest.raises(ValueError):
        page(sh, MinScoreQuery(TermQuery(v[(0, "test")]), -1.0))


# ---------------------------------------------------------------- generated trees: object reference vs compiled arrays

def shadow_nodes(q, sh):
    """test_query_reference.shadow through ConstantScoreQuery and MinScoreQuery"""
    if isinstance(q, ConstantScoreQuery):
        return ConstantScoreQuery(shadow_nodes(q.filter, sh))
    if isinstance(q, MinScoreQuery):
        return MinScoreQuery(shadow_nodes(q.query, sh), q.min_score)
    if isinstance(q, BoostQuery):
        return BoostQuery(shadow_nodes(q.query, sh), q.boost)
    if isinstance(q, BooleanQuery):
        return BooleanQuery([BooleanClause(shadow_nodes(c.query, sh), c.occur) for c in q.clauses], q.minimum_number_should_match)
    if isinstance(q, DisjunctionMaxQuery):
        return DisjunctionMaxQuery([shadow_nodes(d, sh) for d in q.disjuncts], q.tie_breaker)
    return shadow(q, sh)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_generated_trees_equal_the_compiled_judge(built, seed):
    sh = small_shard(seed)
    judge_sh = with_shadow_columns(sh)
    space = qg.space_of(sh, [(0, False), (1, True)], phrase_terms=np.arange(0, 40))
    ref = snr.ScoreNodeReference(sh)
    queries = sg.ScoreNodeGenerator(space, seed, sg.threshold_from(ref)).queries(120)
    nodes = [w for q in queries for w in sg.wrappers(q)]
    assert sum(isinstance(w, ConstantScoreQuery) for w in nodes) > 30 and sum(isinstance(w, MinScoreQuery) for w in nodes) > 30
    k = 50
    want = ref.search(queries, k)
    assert (want[3] > 0).mean() > 0.3
    oix = oracle.OracleIndex(judge_sh)
    got = snr.search(judge_sh, [shadow_nodes(q, sh) for q in queries], k, oix=oix)
    same_pages(got, want, k, queries, seed, "compile_tree + the array-level reference")


def test_generator_reaches_every_depth_and_occur(built):
    sh = small_shard(1)
    space = qg.space_of(sh, [(0, False), (1, True)], phrase_terms=np.arange(0, 40))
    queries = sg.ScoreNodeGenerator(space, 9, sg.threshold_from(snr.ScoreNodeReference(sh))).queries(300)
    seen = set()

    def walk(q, depth, occur, under):
        while isinstance(q, BoostQuery):
            q = q.query
        if isinstance(q, (ConstantScoreQuery, MinScoreQuery)):
            kind = type(q).__name__
            seen.add((kind, "depth", depth))
            seen.add((kind, "occur", occur))
            seen.add((kind, "under", under))
            if isinstance(q, MinScoreQuery):
                seen.add(("threshold", "nan" if math.isnan(q.min_score) else "zero" if q.min_score == 0 else "other"))
            walk(q.filter if isinstance(q, ConstantScoreQuery) else q.query, depth + 1, M, kind)
        elif isinstance(q, BooleanQuery):
            for c in q.clauses:
                walk(c.query, depth + 1, c.occur, "bool")
        elif isinstance(q, DisjunctionMaxQuery):
            for d in q.disjuncts:
                walk(d, depth + 1, S, "dismax")

    for q in queries:
        walk(q, 1, M, "root")
    want = {(k, "depth", d) for k in ("ConstantScoreQuery", "MinScoreQuery") for d in (1, 2, 3)}
    want |= {(k, "occur", o) for k in ("ConstantScoreQuery", "MinScoreQuery") for o in Occur}
    want |= {(k, "under", u) for k in ("ConstantScoreQuery", "MinScoreQuery")
             for u in ("root", "bool", "dismax", "ConstantScoreQuery", "MinScoreQuery")}
    want |= {("threshold", t) for t in ("nan", "zero", "other")}
    assert want <= seen, sorted(map(str, want - seen))
    # every query compiles within the tree limits
    compile_tree([shadow_nodes(q, sh) for q in queries], phrase_table=True)
