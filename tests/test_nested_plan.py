"""Block joins on the host (no GPU): compile_tree's NestedQuery nodes and the product's tree compiler and work planner
(batch_plan.inc compile_tree / plan_work) through the nested planner harness (tests/csrc/nested_plan_harness.cpp) -- the
split into child queries after the request's, the join slots and their scoring flags in every context, the bound of the
child matches, the child pass's work items, and every refusal nrtgpu.h documents for NRTGPU_NODE_NESTED, a lowered join cap
included (NRTGPU_JOIN_CHILDREN itself is read by the context, on the GPU: tests/test_gpu_nested.py)."""
import numpy as np
import pytest

import nested_plan_harness as nj
import plan_harness as ph
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, ConstantScoreQuery, DisjunctionMaxQuery, MinScoreQuery,
                                   NestedQuery, Occur, PhraseQuery, TermQuery, compile_tree)

INVALID, UNSUPPORTED = 1, 3
N_TERMS = 200
N_DOCS = 2_500_000
S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
UNION = -2                 # DevClause.plane of a union / join slot (batch_plan.h kUnionList)
NESTED, TERM, NODE = 6, 0, 3
PATH, PATH2 = 190, 191     # path terms (field 1)
WIDE_SLICE = 1 << 20


@pytest.fixture(scope="module")
def d(built):
    lens = 10 + (np.arange(N_TERMS) * 37) % 500
    lens[PATH], lens[PATH2] = 600_000, 300_000
    off = np.zeros(N_TERMS + 1, np.int64)
    off[1:] = np.cumsum(lens)
    return ph.Dictionary(N_DOCS, off, term_field=np.array([0] * 190 + [1] * 10, np.int32),
                         field_doc_count=np.array([N_DOCS, N_DOCS], np.int64))


def n_post(d, t):
    return int(d.term_off[t + 1] - d.term_off[t])


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(c, o)
    return q


def plan(d, queries, **kw):
    return nj.plan_compiled(d, *compile_tree(queries, phrase_table=True), **kw)


def join_slots(p, q):
    return [c for c in p.query_clauses(q) if c["plane"] == UNION]


def test_compile_tree_kind_6():
    carr, ncl, narr, nn, qarr, nq = compile_tree([BoostQuery(NestedQuery(BoostQuery(TermQuery(3), 2.0), PATH, "avg"), 1.5)])
    kinds = [narr[i].kind for i in range(nn)]
    assert kinds == [NESTED, 0]
    assert narr[0].min_should_match == 1 and narr[0].clause_end - narr[0].clause_begin == 1
    j = carr[narr[0].clause_begin]
    assert j.kind == NODE and j.occur == M and j.id == 1 and j.boost == 1.0
    child = [carr[i] for i in range(narr[1].clause_begin, narr[1].clause_end)]
    assert [(c.occur, c.kind, c.id) for c in child] == [(F, TERM, PATH), (M, TERM, 3)]
    assert child[1].boost == np.float32(np.float32(1.5) * np.float32(2.0))   # the boost folds through the join
    with pytest.raises(ValueError, match="score_mode"):
        compile_tree([NestedQuery(TermQuery(3), PATH, "median")])


def test_split_into_child_queries(d):
    qs = [bq((TermQuery(5), M), (NestedQuery(TermQuery(3), PATH, "sum"), S)),
          NestedQuery(bq((TermQuery(7), S), (TermQuery(8), S)), PATH2, "max"),
          bq((TermQuery(9), S))]
    p = plan(d, qs)
    assert len(p.queries) == 3 + 2 and list(p.join_mode) == [4, 2]
    for j, q in enumerate((0, 1)):
        (slot,) = join_slots(p, q)
        assert p.clauses[p.join_clause[j]]["post_base"] == j and slot["post_base"] == j
        assert slot["kind"] == TERM and slot["n_post"] == 1000   # the parents, as the host's estimate
    assert join_slots(p, 2) == []
    # child query 3: the join's BooleanQuery {FILTER path, MUST 3} is its root
    c3 = p.query_clauses(3)
    assert [(c["occur"], c["post_base"]) for c in c3] == [(F, d.term_off[PATH]), (M, d.term_off[3])]
    assert p.query_nodes(3)[0]["kind"] == 0 and len(p.query_nodes(3)) == 1
    # the parent tree: the join takes a slot and a clause, no node
    assert len(p.query_nodes(0)) == 1 and len(p.query_clauses(0)) == 2
    # work items: the parents' queries only in the parent pass, every child query in every slice in the child pass
    assert set(p.work_query.tolist()) <= {0, 1, 2}
    n_slices = (N_DOCS + WIDE_SLICE - 1) // WIDE_SLICE
    assert sorted(p.join_query.tolist()) == sorted([3, 4] * n_slices)


def test_scoring_flags(d):
    def flags(q, mode="sum"):
        p = plan(d, [q(NestedQuery(bq((TermQuery(3), S), (TermQuery(4), S)), PATH, mode))])
        (slot,) = join_slots(p, 0)
        child = p.query_clauses(1)
        return int(slot["scoring"]), [int(c["scoring"]) for c in child if c["plane"] != UNION and c["occur"] == S]
    assert flags(lambda j: bq((j, M))) == (1, [1, 1])
    assert flags(lambda j: bq((j, S), (TermQuery(5), S))) == (1, [1, 1])
    assert flags(lambda j: bq((j, F))) == (0, [0, 0])
    assert flags(lambda j: bq((j, N), (TermQuery(5), S))) == (0, [0, 0])
    assert flags(lambda j: bq((ConstantScoreQuery(j), M))) == (0, [0, 0])
    # below a MIN_SCORE node everything scores, even inside a CONSTANT node or under FILTER
    assert flags(lambda j: bq((ConstantScoreQuery(MinScoreQuery(j, 0.5)), M))) == (1, [1, 1])
    assert flags(lambda j: bq((MinScoreQuery(j, 0.5), F), (TermQuery(5), S))) == (1, [1, 1])
    assert flags(lambda j: bq((MinScoreQuery(bq((j, F), (TermQuery(5), S)), 0.5), M))) == (0, [0, 0])
    assert flags(lambda j: bq((DisjunctionMaxQuery([j, TermQuery(5)], 0.1), M))) == (1, [1, 1])
    # NONE: the slot scores its entries' 0 where its context scores; the child query only has to match
    assert flags(lambda j: bq((j, M)), "none") == (1, [0, 0])


def test_join_at_depth_and_required_root_slot(d):
    q = bq((bq((bq((NestedQuery(TermQuery(3), PATH, "min"), M), (TermQuery(6), S)), S), (TermQuery(7), S)), M))
    p = plan(d, [q])
    assert len(p.queries) == 2 and len(join_slots(p, 0)) == 1
    p = plan(d, [bq((NestedQuery(TermQuery(3), PATH, "min"), F), (TermQuery(6), S))])
    (slot,) = join_slots(p, 0)
    assert p.queries[0]["req_term_mask"] & (1 << int(slot["slot"]))


def test_bound(d):
    # the child's driver: the rarer of its required lists
    p = plan(d, [NestedQuery(TermQuery(3), PATH, "sum")])
    assert p.join_bound == min(n_post(d, 3), n_post(d, PATH))
    # a disjunction: the sum of its SHOULD lists (the path filter is rarer only when it is below that sum)
    p = plan(d, [NestedQuery(bq((TermQuery(3), S), (TermQuery(4), S)), PATH, "sum")])
    assert p.join_bound == n_post(d, 3) + n_post(d, 4)
    # several joins add up; a phrase drives by its rarest term
    p = plan(d, [NestedQuery(TermQuery(3), PATH, "sum"), bq((NestedQuery(PhraseQuery([10, 11]), PATH, "max"), S))])
    assert p.join_bound == n_post(d, 3) + min(n_post(d, 10), n_post(d, 11))
    # a child query that cannot match is bounded by 0 and has no work items
    p = plan(d, [NestedQuery(bq((TermQuery(3), S), msm=2), PATH, "sum")])
    assert p.join_bound == 0 and len(p.join_query) == 0


def test_refusals(d):
    def err(queries, mutate=None, **kw):
        a = list(compile_tree(queries, phrase_table=True))
        if mutate:
            mutate(a[0], a[2])
        with pytest.raises(ph.PlanError) as e:
            nj.plan_compiled(d, *a, **kw)
        return e.value.rc, e.value.msg

    one = NestedQuery(TermQuery(3), PATH, "sum")

    def set_mode(m):
        def f(carr, narr):
            narr[0].min_should_match = m
        return f

    def second_clause(carr, narr):
        narr[0].clause_end = narr[0].clause_begin + 2

    def not_must(occ):
        def f(carr, narr):
            carr[narr[0].clause_begin].occur = int(occ)
        return f

    assert err([bq((one, M))], set_mode(5)) == (INVALID, "NestedQuery: score mode must be in 0..4")
    assert err([bq((one, M))], set_mode(-1)) == (INVALID, "NestedQuery: score mode must be in 0..4")
    assert err([bq((one, M))], second_clause)[0] == INVALID
    assert "exactly one clause" in err([bq((one, M))], second_clause)[1]
    for occ in (S, F, N):
        assert err([bq((one, M))], not_must(occ)) == (INVALID, "a NestedQuery clause must be MUST")
    assert err([bq((one, M))], n_parents=-1) == (INVALID, "index has no parent docs: nrtgpu_index_add_parents")
    rc, msg = err([NestedQuery(bq((one, S)), PATH, "max")])
    assert rc == UNSUPPORTED and "inside a NestedQuery" in msg
    # tree limits: 8 term slots, 32 clauses in the parent tree ...
    many = bq(*[(TermQuery(20 + i), S) for i in range(8)], (one, S))
    assert err([many])[0] == UNSUPPORTED
    # ... and in a child tree (the path filter takes a slot there)
    assert err([NestedQuery(bq(*[(TermQuery(20 + i), S) for i in range(8)]), PATH, "sum")])[0] == UNSUPPORTED
    # depth: four levels in the child tree counting its root
    deep = bq((bq((bq((TermQuery(3), S)), S)), S))
    plan(d, [NestedQuery(deep, PATH, "sum")])   # root {path, deep}: 4 levels
    assert err([NestedQuery(bq((deep, S)), PATH, "sum")])[0] == UNSUPPORTED
    # ... while the parent tree's depth does not count the child's
    plan(d, [bq((bq((bq((NestedQuery(deep, PATH, "sum"), S)), S)), S))])
    # the join cap
    big = NestedQuery(bq((TermQuery(PATH), S)), PATH2, "sum")
    rc, msg = err([big], max_join_children=100)
    assert rc == UNSUPPORTED and "child matches, more than 100" in msg
    assert plan(d, [big], max_join_children=n_post(d, PATH2)).join_bound == n_post(d, PATH2)

