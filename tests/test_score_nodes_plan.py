"""ConstantScoreQuery and MinScoreQuery nodes on the host (no GPU): compile_tree's node records and boost folding, and the
product's tree compiler (batch_plan.inc compile_tree) through the planner harness -- every refusal with its code and
message, the scoring flags of the clauses below each kind, covers and the driver choice, and the node, level and clause
limits counting the new nodes."""
import ctypes
import math

import numpy as np
import pytest

from nrtsearch_b200 import _native
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, ConstantScoreQuery, DisjunctionMaxQuery, MinScoreQuery, Occur,
                                   PhraseQuery, RangeQuery, TermQuery, compile_tree)
import phrase_plan_harness as pph
import plan_harness as ph
import tree_plan_harness as th
from test_tree_plan import LENS, N_DOCS, _arrays, slots_of

INVALID, UNSUPPORTED = 1, 3
CONSTANT, MIN_SCORE = 3, 4
S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
RANGE = RangeQuery(0, 0, 500_000)
# DevNode of a CONSTANT / MIN_SCORE node: its boost in the tie breaker's word, its threshold in msm's
NODE_VIEW = np.dtype({"names": ["kind", "n_clauses", "n_req", "need_should", "min_score", "boost", "empty"],
                      "formats": ["<i4", "<i4", "<i4", "<i4", "<f4", "<f4", "<i4"],
                      "offsets": [0, 8, 12, 16, 20, 24, 28], "itemsize": 32})


@pytest.fixture(scope="module")
def d(built):
    off = np.zeros(len(LENS) + 1, np.int64)
    off[1:] = np.cumsum(LENS)
    return ph.Dictionary(N_DOCS, off, col_multi=np.array([0, 1], np.uint8), col_n_distinct=np.array([10, 10], np.int32))


def T(t):
    return TermQuery(t)


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(T(c) if isinstance(c, int) else c, o)
    return q


def nodes_of(p, q):
    return p.query_nodes(q).view(NODE_VIEW)


# ---------------------------------------------------------------- compile_tree (Python)

def test_node_records_and_boost_folding():
    f = np.float32
    q = BoostQuery(bq((BoostQuery(ConstantScoreQuery(BoostQuery(T(1), 9.0)), 0.5), S),
                      (BoostQuery(MinScoreQuery(bq((BoostQuery(T(2), 3.0), S)), 0.25), 1.75), M)), 2.0)
    carr, ncl, narr, nn, qarr, nq = compile_tree([q])
    assert nn == 3
    cs, ms, inner = narr[0], narr[1], narr[2]
    assert (cs.kind, ms.kind, inner.kind) == (CONSTANT, MIN_SCORE, 0)
    assert cs.boost == f(f(2.0) * f(0.5)) and ms.boost == f(f(2.0) * f(1.75)) and ms.min_score == f(0.25)
    assert cs.clause_end - cs.clause_begin == 1 and carr[cs.clause_begin].occur == M and carr[cs.clause_begin].id == 1
    assert carr[cs.clause_begin].boost == 9.0                      # the fold starts again below CONSTANT (nothing there scores)
    assert (carr[ms.clause_begin].kind, carr[ms.clause_begin].occur) == (3, M)
    assert carr[inner.clause_begin].boost == 3.0                   # the fold starts again at 1 below MIN_SCORE
    root = [(carr[i].kind, carr[i].id, carr[i].boost) for i in range(qarr[0].clause_begin, qarr[0].clause_end)]
    assert root == [(3, 0, 1.0), (3, 1, 1.0)]


def test_wrappers_at_the_root_and_threshold_zero():
    carr, ncl, narr, nn, qarr, nq = compile_tree([BoostQuery(MinScoreQuery(T(4), 1.5), 3.0), ConstantScoreQuery(T(5))])
    assert nn == 2 and [narr[i].kind for i in range(2)] == [MIN_SCORE, CONSTANT] and narr[0].boost == 3.0
    for i in range(2):
        c = carr[qarr[i].clause_begin]
        assert qarr[i].clause_end - qarr[i].clause_begin == 1 and (c.occur, c.kind, c.id) == (M, 3, i)
    # MinScoreQuery(q, 0) is q, the boosts above it folded into q's leaves (also -0.0)
    for z in (0.0, -0.0):
        a = compile_tree([BoostQuery(MinScoreQuery(BoostQuery(bq((1, S), (2, S)), 0.5), z), 4.0)])
        b = compile_tree([BoostQuery(BoostQuery(bq((1, S), (2, S)), 0.5), 4.0)])
        assert a[3] == b[3] == 0 and bytes(a[0])[:a[1] * 32] == bytes(b[0])[:b[1] * 32]
    carr, ncl, narr, nn, qarr, nq = compile_tree([MinScoreQuery(T(1), math.nan)])
    assert nn == 1 and math.isnan(narr[0].min_score)


def test_python_refusals():
    with pytest.raises(ValueError, match="MinScoreQuery.min_score must be a non-negative number"):
        compile_tree([bq((MinScoreQuery(T(1), -0.5), S))])
    with pytest.raises(ValueError, match="MinScoreQuery.min_score must be a non-negative number"):
        compile_tree([MinScoreQuery(T(1), -math.inf)])
    for b, msg in ((-1.0, "positive"), (math.nan, "finite"), (math.inf, "finite")):
        for q in (BoostQuery(ConstantScoreQuery(T(1)), b), bq((BoostQuery(MinScoreQuery(T(1), 1.0), b), S)),
                  ConstantScoreQuery(BoostQuery(T(1), b))):
            with pytest.raises(ValueError, match=msg):
                compile_tree([q])


def test_six_field_nodes_still_build():
    n = _native.Node(0, 1, 2, 0, 0.5, 0)
    assert (n.kind, n.tie_breaker, n.boost, n.min_score) == (0, 0.5, 0.0, 0.0)
    assert ctypes.sizeof(_native.Node) == 28


# ---------------------------------------------------------------- the product's compiler

# (clauses, nodes, queries, code, message); clauses: occur, kind, id, boost, lo, hi; nodes: kind, begin, end, msm, tie,
# boost, min_score
ROOT = [(1, 3, 0, 1.0, 0, 0)]
Q = [(0, 1, 0, 0, 0, 0.0)]
REFUSED = [
    (ROOT + [(1, 0, 1, 1.0, 0, 0)], [(2, 1, 2, 0, 0.0, 1.0, 0.0)], "bad node kind"),
    (ROOT + [(1, 0, 1, 1.0, 0, 0)], [(5, 1, 2, 0, 0.0, 1.0, 0.0)], "bad node kind"),
    (ROOT + [(1, 0, 1, 1.0, 0, 0)], [(CONSTANT, 1, 1, 0, 0.0, 1.0, 0.0)], "exactly one clause"),
    (ROOT + [(1, 0, 1, 1.0, 0, 0)], [(MIN_SCORE, 1, 1, 0, 0.0, 1.0, 1.0)], "exactly one clause"),
    (ROOT + [(1, 0, 1, 1.0, 0, 0), (1, 0, 2, 1.0, 0, 0)], [(CONSTANT, 1, 3, 0, 0.0, 1.0, 0.0)], "exactly one clause"),
    (ROOT + [(1, 0, 1, 1.0, 0, 0), (1, 0, 2, 1.0, 0, 0)], [(MIN_SCORE, 1, 3, 0, 0.0, 1.0, 1.0)], "exactly one clause"),
    (ROOT + [(0, 0, 1, 1.0, 0, 0)], [(CONSTANT, 1, 2, 0, 0.0, 1.0, 0.0)], "clause must be MUST"),
    (ROOT + [(2, 0, 1, 1.0, 0, 0)], [(MIN_SCORE, 1, 2, 0, 0.0, 1.0, 1.0)], "clause must be MUST"),
    (ROOT + [(3, 0, 1, 1.0, 0, 0)], [(CONSTANT, 1, 2, 0, 0.0, 1.0, 0.0)], "clause must be MUST"),
    (ROOT + [(1, 0, 1, 1.0, 0, 0)], [(MIN_SCORE, 1, 2, 0, 0.0, 1.0, -1.0)], "MinScoreQuery.min_score must be a non-negative number"),
    (ROOT + [(1, 0, 1, 1.0, 0, 0)], [(MIN_SCORE, 1, 2, 0, 0.0, 1.0, -math.inf)], "MinScoreQuery.min_score must be a non-negative number"),
]
for kind in (CONSTANT, MIN_SCORE):
    for b, msg in ((-1.0, "Boost must be a positive number"), (math.nan, "Boost must be a finite number"),
                   (math.inf, "Boost must be a finite number")):
        REFUSED.append((ROOT + [(1, 0, 1, 1.0, 0, 0)], [(kind, 1, 2, 0, 0.0, b, 1.0)], msg))


@pytest.mark.parametrize("clauses,nodes,msg", REFUSED)
def test_refusals(d, clauses, nodes, msg):
    with pytest.raises(ph.PlanError) as e:
        th.plan_compiled(d, *_arrays(clauses, nodes, Q), 10)
    assert e.value.rc == INVALID and msg in e.value.msg, e.value.msg


def test_accepted_edges(d):
    """a NaN threshold, 0, and boosts of 0 and the largest float compile; BOOL and DISMAX ignore the new words"""
    for nd in ((MIN_SCORE, 1, 2, 0, 0.0, 0.0, math.nan), (MIN_SCORE, 1, 2, 0, 0.0, 3.4028235e38, 0.0),
               (CONSTANT, 1, 2, 0, 0.0, 0.0, -1.0), (0, 1, 2, 0, 0.0, -1.0, -1.0), (1, 1, 2, 0, 0.5, math.nan, -1.0)):
        occ = 0 if nd[0] == 1 else 1
        p = th.plan_compiled(d, *_arrays(ROOT + [(occ, 0, 1, 1.0, 0, 0)], [nd], Q), 10)
        n = nodes_of(p, 0)[1]
        if nd[0] in (CONSTANT, MIN_SCORE):
            assert np.float32(nd[5]).tobytes() == n["boost"].tobytes()
        if nd[0] == MIN_SCORE:
            assert np.float32(nd[6]).tobytes() == n["min_score"].tobytes()


def test_scoring_flags(d):
    # root: SHOULD CONSTANT(bool(t0, t1 MUST)), FILTER MIN_SCORE(t2), MUST_NOT CONSTANT(MIN_SCORE(bool(t3 S, phrase-free)))
    q = bq((ConstantScoreQuery(bq((0, S), (1, M))), S), (MinScoreQuery(T(2), 1.0), F),
           (ConstantScoreQuery(MinScoreQuery(bq((3, S), (RANGE, S)), 2.0)), N), (4, S))
    p = th.plan(d, [q], 10)
    cl = p.query_clauses(0)
    nodes = nodes_of(p, 0)
    assert list(nodes["kind"]) == [0, CONSTANT, 0, MIN_SCORE, CONSTANT, MIN_SCORE, 0]
    # the node of each leaf, the child of each node clause: the "pad_" word (DevClause::node)
    leaves = [(int(c["pad_"]), int(c["kind"]), int(c["scoring"])) for c in cl if c["kind"] != 3]
    node_clauses = [(int(c["pad_"]), int(c["scoring"])) for c in cl if c["kind"] == 3]
    # root leaves: t4 SHOULD scores
    assert (0, 0, 1) in leaves
    # below CONSTANT (node 1): its bool clause (node 2) does not score, nor t0 / t1 in node 2
    assert [(n, s) for n, k, s in leaves if n == 2] == [(2, 0), (2, 0)]
    # MIN_SCORE under FILTER (node 3): its term scores
    assert [(n, k, s) for n, k, s in leaves if n == 3] == [(3, 0, 1)]
    # MIN_SCORE (node 5) under CONSTANT (node 4) under MUST_NOT: the bool below it (node 6) scores
    assert [(n, k, s) for n, k, s in leaves if n == 6] == [(6, 0, 1), (6, 1, 1)]
    # the node clauses: root -> 1 (SHOULD, scores), root -> 3 (FILTER), root -> 4 (MUST_NOT), 1 -> 2 (not), 3: none,
    # 4 -> 5 (below CONSTANT: no), 5 -> 6 (below MIN_SCORE: yes)
    assert node_clauses == [(1, 1), (3, 0), (4, 0), (2, 0), (5, 0), (6, 1)]
    assert [int(n["n_req"]) for n in nodes[[1, 3, 4, 5]]] == [1] * 4 and (nodes["need_should"][[1, 3, 4, 5]] == 0).all()
    assert nodes["boost"][1] == 1.0 and nodes["min_score"][3] == 1.0 and nodes["min_score"][5] == 2.0


def test_phrase_below_min_score_scores(d):
    """a phrase leaf below MIN_SCORE is compiled scoring (all its matches counted), below CONSTANT presence-only"""
    qs = [MinScoreQuery(PhraseQuery([1, 2]), 1.0), ConstantScoreQuery(PhraseQuery([1, 2])),
          bq((MinScoreQuery(PhraseQuery([1, 2]), 1.0), F))]
    p = pph.plan_compiled(d, *compile_tree(qs, phrase_table=True))
    for q, want in zip(range(3), (1, 0, 1)):
        phr = [c for c in p.query_clauses(q) if c["kind"] == 4]
        assert len(phr) == 1 and int(phr[0]["scoring"]) == want, q


def test_covers_and_driver(d):
    # a wrapper is covered by its clause: MUST CONSTANT(t4 (1000)) vs MUST MIN_SCORE(t5 | t6 (75)): the cheaper one leads
    p = th.plan(d, [bq((ConstantScoreQuery(T(4)), M), (MinScoreQuery(bq((5, S), (6, S)), 0.5), M))], 10)
    assert p.queries[0]["driver_mask"] == slots_of(p, 0, [5, 6]) and not p.queries[0]["dense_driver"]
    # at the root, over a term: that term drives
    p = th.plan(d, [MinScoreQuery(T(3), 2.0), ConstantScoreQuery(T(7))], 10)
    assert p.queries[0]["driver_mask"] == slots_of(p, 0, [3]) and p.queries[1]["driver_mask"] == slots_of(p, 1, [7])
    # SHOULD wrappers unite into the root's cover
    p = th.plan(d, [bq((ConstantScoreQuery(T(0)), S), (BoostQuery(MinScoreQuery(T(1), 1.0), 2.0), S))], 10)
    assert p.queries[0]["driver_mask"] == slots_of(p, 0, [0, 1])
    # over a range: no cover, the dense driver
    p = th.plan(d, [ConstantScoreQuery(RANGE), bq((MinScoreQuery(RANGE, 1.0), S), (2, S))], 10)
    assert list(p.queries["dense_driver"]) == [1, 1] and list(p.queries["driver_mask"]) == [0, 0]
    # can match iff the clause can
    p = th.plan(d, [ConstantScoreQuery(bq((0, S), msm=2)), bq((MinScoreQuery(DisjunctionMaxQuery([], 0.0), 1.0), S), (2, S)),
                    MinScoreQuery(bq((0, S), (1, S), msm=2), 1.0)], 10)
    assert list(p.queries["empty"]) == [1, 0, 0]
    assert p.queries[1]["driver_mask"] == slots_of(p, 1, [2])
    assert set(p.work_query) == {1, 2}


def test_limits_count_the_new_nodes(d):
    eight = bq(*[(ConstantScoreQuery(T(t)) if t % 2 else MinScoreQuery(T(t), 1.0), S) for t in range(8)])
    th.plan(d, [eight], 10)
    with pytest.raises(ph.PlanError) as e:
        th.plan(d, [bq(*[(ConstantScoreQuery(T(t)), S) for t in range(8)], (ConstantScoreQuery(RANGE), S))], 10)
    assert e.value.rc == UNSUPPORTED and "nested" in e.value.msg
    deep4 = ConstantScoreQuery(MinScoreQuery(ConstantScoreQuery(T(0)), 1.0))   # root + 3 wrappers: 4 levels
    th.plan(d, [deep4], 10)
    with pytest.raises(ph.PlanError) as e:
        th.plan(d, [MinScoreQuery(deep4, 1.0)], 10)
    assert e.value.rc == UNSUPPORTED and "4 levels" in e.value.msg
    # 32 clauses: 15 wrappers' node clauses and their 15 range clauses + 2 more
    fifteen = [(ConstantScoreQuery(RANGE), S)] * 7 + [(RANGE, S)] * 17
    th.plan(d, [bq(*fifteen)], 10)   # 7 node clauses + 7 wrapped + 17 = 31
    with pytest.raises(ph.PlanError) as e:
        th.plan(d, [bq(*fifteen, (RANGE, S), (RANGE, S))], 10)
    assert e.value.rc == UNSUPPORTED and "32 clauses" in e.value.msg
