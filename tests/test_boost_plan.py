"""Boost refusals on the host (no GPU): a NaN or infinite boost is refused by both Python query compilers
(compile_queries, compile_tree) and by the product's compiler (batch_plan.inc compile_batch, flat and tree clause paths)
through the planner harness, as a negative one is. Such a boost would make a NaN or infinite BM25 weight and scores with
no place in the (score desc, doc asc) order."""
import numpy as np
import pytest

from nrtsearch_b200 import _native
from nrtsearch_b200.search import BooleanQuery, BoostQuery, Occur, RangeQuery, TermQuery, compile_queries, compile_tree
import plan_harness as ph
import tree_plan_harness as th

INVALID = 1
NAN, INF = float("nan"), float("inf")
S, M = Occur.SHOULD, Occur.MUST


@pytest.fixture(scope="module")
def d(built):
    off = np.concatenate([[0], np.cumsum([100, 200, 300, 50])]).astype(np.int64)
    return ph.Dictionary(1_000_000, off, col_multi=np.array([0, 1], np.uint8), col_n_distinct=np.array([10, 10], np.int32))


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(TermQuery(c) if isinstance(c, int) else c, o)
    return q


@pytest.mark.parametrize("b", [NAN, INF, -INF])
def test_python_compilers_refuse_non_finite_boosts(b):
    """at the root, around a node, around a leaf and inside nested BoostQuerys"""
    for q in (BoostQuery(bq((1, S)), b), bq((BoostQuery(bq((1, S)), 2.0), M), (BoostQuery(TermQuery(2), b), S)),
              bq((BoostQuery(BoostQuery(bq((1, S), (2, S)), b), 0.5), M))):
        with pytest.raises(ValueError, match="Boost must be a"):
            compile_tree([q])
    for q in (BoostQuery(bq((1, S)), b), bq((BoostQuery(BoostQuery(TermQuery(2), 0.5), b), S)), BoostQuery(RangeQuery(0, 0, 9), b)):
        with pytest.raises(ValueError, match="Boost must be a"):
            compile_queries([q])


def _arrays(clauses, nodes, queries):
    carr = (_native.Clause * max(len(clauses), 1))(*[_native.Clause(*c) for c in clauses])
    narr = (_native.Node * max(len(nodes), 1))(*[_native.Node(*n) for n in nodes])
    qarr = (_native.Query * len(queries))(*[_native.Query(*q) for q in queries])
    return carr, len(clauses), narr, len(nodes), qarr, len(queries)


# (clauses, nodes, queries, message); clauses: occur, kind, id, boost, lo, hi. Without nodes the flat path compiles them.
NON_FINITE = [
    ([(1, 0, 1, NAN, 0, 0)], [], [(0, 1, 0, 0, 0, 0.0)], "Boost must be a finite number"),                 # flat term
    ([(0, 0, 1, 1.0, 0, 0), (2, 1, 0, INF, 0, 10)], [], [(0, 2, 0, 0, 0, 0.0)], "Boost must be a finite number"),  # flat range
    ([(0, 2, 0, INF, 0, 0)], [], [(0, 1, 0, 0, 0, 0.0)], "Boost must be a finite number"),                 # flat match-all
    ([(1, 3, 0, 1.0, 0, 0), (0, 0, 1, NAN, 0, 0)], [(0, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "Boost must be a finite number"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 2, 0, INF, 0, 0)], [(1, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "Boost must be a finite number"),
    ([(1, 3, 0, 1.0, 0, 0), (0, 0, 1, -INF, 0, 0)], [(0, 1, 2, 0, 0.0, 0)], [(0, 1, 0, 0, 0, 0.0)], "Boost must be a positive number"),
    ([(1, 0, 1, 1.0, 0, 0), (0, 0, 2, NAN, 0, 0)], [], [(0, 1, 0, 0, 0, 0.0), (1, 2, 0, 0, 0, 0.0)], "Boost must be a finite number"),
]


@pytest.mark.parametrize("case", range(len(NON_FINITE)))
def test_product_compiler_refuses_non_finite_boosts(d, case):
    clauses, nodes, queries, msg = NON_FINITE[case]
    with pytest.raises(ph.PlanError) as e:
        th.plan_compiled(d, *_arrays(clauses, nodes, queries), 10)
    assert e.value.rc == INVALID and msg in e.value.msg, e.value.msg


def test_finite_boosts_still_compile(d):
    """the edges of the finite domain: 0, the smallest subnormal, the largest float"""
    for b in (0.0, 2.0**-149, float(np.finfo(np.float32).max)):
        th.plan_compiled(d, *_arrays([(1, 0, 1, b, 0, 0)], [], [(0, 1, 0, 0, 0, 0.0)]), 10)
        th.plan_compiled(d, *_arrays([(1, 3, 0, 1.0, 0, 0), (0, 0, 1, b, 0, 0)], [(0, 1, 2, 0, 0.0, 0)],
                                     [(0, 1, 0, 0, 0, 0.0)]), 10)
