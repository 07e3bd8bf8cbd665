"""Query trees on the host (no GPU): compile_tree's layout and refusals, and the product's tree compiler and work planner
(batch_plan.inc compile_tree, plan_work) through the planner harness -- covers, dense drivers, emptiness, the wide choice
and every refusal nrtgpu_search_tree documents."""
import numpy as np
import pytest

from nrtsearch_b200 import NrtGpuUnsupported, _native
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, MatchAllDocsQuery, Occur, RangeQuery, TermQuery,
                                   compile_queries, compile_tree)
import plan_harness as ph
import tree_plan_harness as th

INVALID, UNSUPPORTED = 1, 3
LENS = [100, 200, 300, 50, 1000, 5, 70, 80, 90, 110]   # postings of terms 0..9
N_DOCS = 3_000_000


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


S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
RANGE = RangeQuery(0, 0, 500_000)


def slots_of(p, q, terms):
    """driver mask of the term ids `terms` in query q's compiled clauses"""
    cl = p.query_clauses(q)
    slot = {}
    for c in cl:
        if c["kind"] == 0:
            slot.setdefault(int(c["post_base"]), int(c["slot"]))
    off = np.concatenate([[0], np.cumsum(LENS)])
    return sum(1 << slot[int(off[t])] for t in terms)


# ---------------------------------------------------------------- compile_tree (Python mirror)

def test_compile_tree_layout_preorder_and_folded_boosts():
    inner = bq((0, S), (BoostQuery(T(1), 3.0), S))
    dm = DisjunctionMaxQuery([bq((2, S), (3, S)), T(4)], 0.3)
    q = BoostQuery(bq((BoostQuery(inner, 0.5), M), (dm, S), (RANGE, F), msm=1), 2.0)
    carr, ncl, narr, nn, qarr, nq = compile_tree([q, T(7)])
    assert (nq, nn) == (2, 3)
    # root clauses first, then the nodes in pre-order: inner (0), the dismax (1), the dismax's bool (2)
    root = [(carr[i].occur, carr[i].kind, carr[i].id, carr[i].boost) for i in range(qarr[0].clause_begin, qarr[0].clause_end)]
    assert root == [(M, 3, 0, 1.0), (S, 3, 1, 1.0), (F, 1, 0, 2.0)]
    assert qarr[0].min_should_match == 1
    n0, n1, n2 = narr[0], narr[1], narr[2]
    assert (n0.kind, n1.kind, n2.kind) == (0, 1, 0)
    assert abs(n1.tie_breaker - 0.3) < 1e-7
    leaves0 = [(carr[i].kind, carr[i].id, carr[i].boost) for i in range(n0.clause_begin, n0.clause_end)]
    assert leaves0 == [(0, 0, 1.0), (0, 1, float(np.float32(np.float32(2.0) * np.float32(0.5)) * np.float32(3.0)))]
    d1 = [(carr[i].kind, carr[i].id, carr[i].occur) for i in range(n1.clause_begin, n1.clause_end)]
    assert d1 == [(3, 2, S), (0, 4, S)]
    assert [carr[i].id for i in range(n2.clause_begin, n2.clause_end)] == [2, 3]
    assert all(carr[i].boost == 2.0 for i in range(n2.clause_begin, n2.clause_end))
    # a bare leaf root: one MUST clause, as compile_queries
    assert (qarr[1].clause_end - qarr[1].clause_begin, carr[qarr[1].clause_begin].occur) == (1, M)


def test_compile_tree_dismax_root_is_one_must_node():
    carr, ncl, narr, nn, qarr, nq = compile_tree([DisjunctionMaxQuery([T(1), T(2)], 0.5)])
    assert nn == 1 and qarr[0].clause_end - qarr[0].clause_begin == 1
    c = carr[qarr[0].clause_begin]
    assert (c.occur, c.kind, c.id) == (M, 3, 0) and narr[0].kind == 1


def test_compile_tree_of_flat_queries_matches_compile_queries():
    qs = [bq((1, S), (2, S), msm=1), BoostQuery(bq((3, M), (RANGE, F)), 1.5), MatchAllDocsQuery()]
    a = compile_queries(qs)
    carr, ncl, narr, nn, qarr, nq = compile_tree(qs)
    assert nn == 0 and ncl == a[1] and nq == a[3]
    assert bytes(carr)[:ncl * 32] == bytes(a[0])[:ncl * 32] and bytes(qarr) == bytes(a[2])


def test_compile_tree_refusals():
    with pytest.raises(ValueError, match="Boost must be a positive number"):
        compile_tree([bq((BoostQuery(bq((1, S)), -1.0), M))])
    with pytest.raises(NrtGpuUnsupported):
        compile_tree([bq((object(), M))])
    with pytest.raises(NrtGpuUnsupported, match="nested BooleanQuery"):
        compile_queries([bq((bq((1, S)), M))])


# ---------------------------------------------------------------- compile_tree (product) through the planner harness

def test_tree_batch_is_wide_with_one_item_per_query_and_slice(d):
    p = th.plan(d, [bq((bq((0, S), (1, S)), M), (RANGE, F)), bq((2, S), (3, S))], 10)
    assert p.tree and p.wide and p.n_slices == -(-N_DOCS // ph.constants()["kWideSliceDocs"])
    assert p.n_work == 2 * p.n_slices and p.n_probe_simple == p.n_probe_generic == 0


def test_flat_request_is_unchanged_without_node_clauses(d):
    qs = [bq((1, S), (2, S)), bq((3, M), (RANGE, F))]
    flat = ph.plan(d, qs, 10)
    p = th.plan(d, qs, 10)
    assert not p.tree and not p.wide
    assert p.counters == flat.counters and p.clauses.tobytes() == flat.clauses.tobytes() and p.queries.tobytes() == flat.queries.tobytes()


def test_match_in_bool_is_driven_by_its_should_terms(d):
    p = th.plan(d, [bq((bq((0, S), (1, S)), M), (RANGE, F))], 10)
    q = p.queries[0]
    assert not q["dense_driver"] and q["driver_mask"] == slots_of(p, 0, [0, 1]) and not q["empty"]
    nodes = p.query_nodes(0)
    assert len(nodes) == 2 and nodes[0]["n_req"] == 2 and nodes[1]["need_should"] == 1


def test_cheapest_required_cover(d):
    # MUST t4 (1000 postings) vs MUST (t5 | t6) (75): the node's union is cheaper
    p = th.plan(d, [bq((4, M), (bq((5, S), (6, S)), M))], 10)
    assert p.queries[0]["driver_mask"] == slots_of(p, 0, [5, 6]) and p.queries[0]["has_non_driver"]
    # ... and MUST t3 (50) beats it
    p = th.plan(d, [bq((bq((5, S), (6, S)), M), (3, F))], 10)
    assert p.queries[0]["driver_mask"] == slots_of(p, 0, [3])


def test_should_union_and_dismax_union(d):
    p = th.plan(d, [bq((bq((0, M), (1, M)), S), (DisjunctionMaxQuery([T(2), bq((3, S), (4, S))], 0.2), S))], 10)
    # first node: cheapest required (t0); dismax: union of t2 and (t3 | t4)
    assert p.queries[0]["driver_mask"] == slots_of(p, 0, [0, 2, 3, 4])


def test_no_cover_takes_the_dense_driver(d):
    qs = [bq((bq((0, S), (RANGE, S)), M)),                 # a SHOULD range: the node has no cover
          bq((bq((RANGE, M), (1, S)), M)),                 # need_should 0 and a range required: none
          bq((DisjunctionMaxQuery([T(1), MatchAllDocsQuery()], 0.0), M)),
          bq((bq((0, S)), S), (RANGE, S))]                 # a SHOULD range at the root
    p = th.plan(d, qs, 10)
    for q in range(len(qs)):
        assert p.queries[q]["dense_driver"] == 1 and p.queries[q]["driver_mask"] == 0, q
    # a required term rescues the node with a range
    p = th.plan(d, [bq((bq((RANGE, M), (1, S)), M), (2, M))], 10)
    assert not p.queries[0]["dense_driver"] and p.queries[0]["driver_mask"] == slots_of(p, 0, [2])


def test_emptiness_propagates(d):
    qs = [bq((bq((0, S), (1, S), msm=3), M), (2, S)),     # msm above the node's SHOULD count, required: the root is empty
          bq((bq((0, N), (1, N)), F), (2, S)),            # all-MUST_NOT node, required
          bq((bq((0, S), msm=2), S), (2, S)),             # empty SHOULD node: the root is not empty, covered by t2
          bq((DisjunctionMaxQuery([], 0.0), M)),          # dismax of nothing
          bq((bq((bq((0, S), msm=2), S)), S)),            # only SHOULD child empty -> empty, one level up
          bq((bq((bq((0, S), msm=2), M), (1, S)), S), (3, S))]
    p = th.plan(d, qs, 10)
    assert list(p.queries["empty"]) == [1, 1, 0, 1, 1, 0]
    assert p.queries[2]["driver_mask"] == slots_of(p, 2, [2])
    assert p.queries[5]["driver_mask"] == slots_of(p, 5, [3])    # the first SHOULD node is empty: covered by nothing
    assert set(p.work_query) == {2, 5} and p.n_work == 2 * p.n_slices   # empty roots get no work items
    n1 = p.query_nodes(1)
    assert n1[1]["empty"] == 1 and n1[0]["empty"] == 1


def test_scoring_flags_and_parents(d):
    p = th.plan(d, [bq((bq((0, S), (1, S)), F), (bq((2, M), (bq((3, S)), N)), M), (4, S))], 10)
    cl = p.query_clauses(0)
    nodes = p.query_nodes(0)
    assert len(nodes) == 4
    # root clauses: node, node, t4; then node 1 (t0, t1), node 2 (t2, node 3), node 3 (t3)
    assert list(cl["kind"]) == [3, 3, 0, 0, 0, 0, 3, 0]
    assert list(cl["pad_"]) == [1, 2, 0, 1, 1, 2, 3, 3]   # child of a node clause, node of a leaf
    assert list(cl["scoring"]) == [0, 1, 1, 0, 0, 1, 0, 0]
    assert [int(n["clause_begin"]) for n in nodes] == [0, 3, 5, 7]


def test_tree_limits(d):
    eight = bq(*[(bq((t, S)), S) for t in range(8)])
    th.plan(d, [eight], 10)   # 8 nested nodes, 8 term leaves
    with pytest.raises(ph.PlanError) as e:
        th.plan(d, [bq(*[(bq((t, S)), S) for t in range(9)])], 10)
    assert e.value.rc == UNSUPPORTED and "nested" in e.value.msg
    with pytest.raises(ph.PlanError) as e:
        th.plan(d, [bq((bq(*[(t, S) for t in range(9)]), M))], 10)
    assert e.value.rc == UNSUPPORTED and "8 term leaves" in e.value.msg
    with pytest.raises(ph.PlanError) as e:
        th.plan(d, [bq((bq(*[(RANGE, S)] * 31), M), (RANGE, S))], 10)
    assert e.value.rc == UNSUPPORTED and "32 clauses" in e.value.msg
    th.plan(d, [bq((bq(*[(RANGE, S)] * 30), M), (RANGE, S))], 10)   # 32 clauses
    deep4 = bq((bq((bq((bq((0, S)), M)), M)), M))
    th.plan(d, [deep4], 10)
    with pytest.raises(ph.PlanError) as e:
        th.plan(d, [bq((deep4, M))], 10)
    assert e.value.rc == UNSUPPORTED and "4 levels" in e.value.msg
    with pytest.raises(ph.PlanError) as e:
        th.plan(d, [deep4], 1025)
    assert e.value.rc == UNSUPPORTED and "top_k" in e.value.msg
    p = th.plan(d, [deep4], 1024)
    assert p.wide


def _arrays(clauses, nodes, queries):
    carr = (_native.Clause * max(len(clauses), 1))(*[_native.Clause(*c) for c in clauses])
    narr = (_native.Node * max(len(nodes), 1))(*[_native.Node(*n) for n in nodes])
    qarr = (_native.Query * len(queries))(*[_native.Query(*q) for q in queries])
    return carr, len(clauses), narr, len(nodes), qarr, len(queries)


# (clauses, nodes, queries, message) of every INVALID tree (clauses: occur, kind, id, boost, lo, hi)
INVALID_TREES = [
    ([(1, 3, 1, 1.0, 0, 0)], [(0, 0, 0, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "node id out of range"),
    ([(1, 3, -1, 1.0, 0, 0)], [(0, 0, 0, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "node id out of range"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 3, 0, 1.0, 0, 0)], [(0, 2, 2, 0, 0.0, 0)], [(0, 2, 0, 0, 0, 0.0)], "more than once"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 3, 0, 1.0, 0, 0)], [(0, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "more than once or from a cycle"),
    ([(1, 3, 0, 1.0, 0, 0), (1, 0, 1, 1.0, 0, 0)], [(1, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "must be SHOULD"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 0, 1, 1.0, 0, 0)], [(1, 1, 2, 0, 1.5, 0)], [(0, 1, 0, 0, 0, 0.0)], "tieBreakerMultiplier"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 0, 1, 1.0, 0, 0)], [(1, 1, 2, 0, -0.1, 0)], [(0, 1, 0, 0, 0, 0.0)], "tieBreakerMultiplier"),
    ([(1, 3, 0, 2.0, 0, 0), (0, 0, 1, 1.0, 0, 0)], [(0, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "boost 1"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 0, 1, 1.0, 0, 0)], [(2, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "bad node kind"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 0, 1, 1.0, 0, 0)], [(0, 1, 3, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "node clause range"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 0, 1, 1.0, 0, 0)], [(0, 1, 2, -1, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "minimumNumberShouldMatch"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 0, 2_000_000_000, 1.0, 0, 0)], [(0, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "term id out of range"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 1, 5, 1.0, 0, 0)], [(0, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "column id out of range"),
    ([(1, 3, 0, 1.0, 0, 0), (4, 0, 1, 1.0, 0, 0)], [(0, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "bad occur"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 0, 1, -1.0, 0, 0)], [(0, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "Boost must be a positive"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 7, 1, 1.0, 0, 0)], [(0, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "bad clause kind"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 0, 1, 1.0, 0, 0)], [(0, 1, 2, 0, 0.0, 0)], [(0, 3, 0, 0, 0, 0.0)], "out of bounds"),
]


@pytest.mark.parametrize("clauses,nodes,queries,msg", INVALID_TREES)
def test_invalid_trees(d, clauses, nodes, queries, msg):
    with pytest.raises(ph.PlanError) as e:
        th.plan_compiled(d, *_arrays(clauses, nodes, queries), 10)
    assert e.value.rc == INVALID and msg in e.value.msg, e.value.msg


def test_node_clauses_need_nodes(d):
    """Without nodes a node clause is a bad clause kind (every existing entry point)"""
    with pytest.raises(ph.PlanError) as e:
        th.plan_compiled(d, *_arrays([(1, 3, 0, 1.0, 0, 0)], [], [(0, 1, 0, 0, 0, 0.0)]), 10)
    assert e.value.rc == INVALID and "bad clause kind" in e.value.msg


def test_sorted_and_aggregations_on_a_tree_are_unsupported(d):
    tree = [bq((bq((0, S), (1, S)), M))]
    with pytest.raises(ph.PlanError) as e:
        th.plan(d, tree, 10, sort=_native.Sort(1, 0, 0, 0, 0, None))
    assert e.value.rc == UNSUPPORTED
    with pytest.raises(ph.PlanError) as e:
        th.plan(d, tree, 10, aggs=[_native.Aggregation(2, 0, 0, 0, 0, 0)])
    assert e.value.rc == UNSUPPORTED


def test_search_after_key_as_flat(d):
    from nrtsearch_b200.search import ScoreDoc
    p = th.plan(d, [bq((bq((0, S), (1, S)), M))], 10, search_after=[ScoreDoc(123, 2.5)])
    flat = ph.plan(d, [bq((0, S), (1, S))], 10, search_after=[ScoreDoc(123, 2.5)])
    assert p.queries[0]["has_after"] == 1 and p.queries[0]["after_key"] == flat.queries[0]["after_key"]
