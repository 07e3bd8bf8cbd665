"""The collector rules of the host batch compiler for nrtgpu_search_tree_aggs, on the CPU through
tests/csrc/window_aggs_plan_harness.cpp: with window_collectors set, a query tree, a phrase batch or a wide flat batch with
collectors compiles for the window engine with an exact threshold and its collectors recorded; a narrow flat batch compiles
exactly as the flat aggregation request does; every other collector rule still refuses. Without the field the refusals of
the existing entry points hold. CPU only."""
import ctypes as C

import numpy as np
import pytest

import plan_harness as ph
import window_aggs_plan_harness as wh
from nrtsearch_b200 import _native
from nrtsearch_b200._native import AggFilter, Aggregation as A, NestedAggregation as N, NestedSort
from nrtsearch_b200.search import BooleanQuery, DisjunctionMaxQuery, MatchAllDocsQuery, Occur, PhraseQuery, RangeQuery, TermQuery

INVALID, UNSUPPORTED = 1, 3
TERMS, MIN, MAX, SUM, TOP_HITS, FILTER = 1, 2, 3, 4, 5, 6
S, M, F, N_ = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
LENS = [100, 200, 300, 50, 1000, 5, 70, 80, 90, 110]   # postings of terms 0..9
N_DOCS = 3_000_000
ORDER = (C.c_void_p * 1)(0x1000)   # opaque to the compiler: any address stands for an order
SORTED, NONE = NestedSort(C.cast(ORDER, C.c_void_p), None), NestedSort()


@pytest.fixture(scope="module")
def d(built):
    off = np.zeros(len(LENS) + 1, np.int64)
    off[1:] = np.cumsum(LENS)
    # column 0: single-valued, 10 values; column 1: multi-valued; column 2: single-valued, 1M values
    return ph.Dictionary(N_DOCS, off, col_multi=np.array([0, 1, 0], np.uint8), col_n_distinct=np.array([10, 10, 1_000_000], np.int32))


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(TermQuery(c) if isinstance(c, int) else c, o)
    return q


def terms(col=0, size=10, filter_agg=0):
    return A(TERMS, col, 0, size, 1, filter_agg)


def top(parent, hits=3, start=0):
    return N(parent, TOP_HITS, 0, 0, hits, start, 0, 0)


TREES = [
    bq((bq((0, S), (1, S)), M), (RangeQuery(0, 0, 500_000), F)),
    bq((DisjunctionMaxQuery([bq((2, S), (3, S)), TermQuery(4)], 0.3), M), (5, N_)),
    bq((PhraseQuery([6, 7], slop=1), M), (MatchAllDocsQuery(), S)),
]
COLLECTORS = dict(aggs=[terms(0), A(MAX, 2, 0, 0, 0, 0), A(FILTER, 0, 0, 0, 0, 0), terms(2, 5, 3)],
                  nested=[top(0), N(0, SUM, 2, 0, 0, 0, 1, 0), top(2, 4, 1), N(2, MIN, 0, 0, 0, 0, 0, 0)],
                  nested_sorts=[SORTED, NONE, NONE, NONE],
                  filters=[AggFilter(), AggFilter(), AggFilter(1, 0, 0, 0, None), AggFilter()],
                  filter_queries=[bq((8, S), (9, S))])


def test_tree_with_collectors_compiles_for_the_window_engine(d):
    p = wh.plan(d, TREES, 10, **COLLECTORS)
    assert p.tree and p.wide and p.n_probe_simple == p.n_probe_generic == 0
    assert p.n_work == len(TREES) * p.n_slices and p.n_phrases == 1
    assert p.threshold == ph.INT_MAX
    assert (p.n_aggs, p.n_nested, p.n_sorted, p.n_filters, p.agg_filter_queries) == (4, 4, 1, 1, 1)
    assert [(p.aggs[i].kind, p.aggs[i].column, p.aggs[i].filter_agg) for i in range(4)] == [(1, 0, 0), (3, 2, 0), (6, 0, 0), (1, 2, 3)]
    assert [(p.nested[j].parent, p.nested[j].kind, p.nested[j].top_hits) for j in range(4)] == [(0, 5, 3), (0, 4, 0), (2, 5, 4), (2, 2, 0)]


def test_tree_without_the_field_keeps_its_refusal(d):
    with pytest.raises(ph.PlanError) as e:
        wh.plan(d, TREES, 10, window_collectors=False, **COLLECTORS)
    assert e.value.rc == UNSUPPORTED and e.value.msg == "aggregations over a query tree are not on the GPU path"


@pytest.mark.parametrize("shape", ["six_terms", "top_k_1024"])
def test_wide_flat_batch_with_collectors(d, shape):
    if shape == "six_terms":
        qs, k = [bq(*[(t, S) for t in range(6)]), bq((0, M), (1, S))], 10
    else:
        qs, k = [bq((0, S), (1, S)), bq((2, M), (3, M))], 1024
    p = wh.plan(d, qs, k, aggs=[terms(0)], nested=[top(0)])
    assert p.wide and not p.tree and p.n_work == len(qs) * p.n_slices and p.threshold == ph.INT_MAX
    assert p.n_aggs == 1 and p.n_nested == 1
    with pytest.raises(ph.PlanError) as e:
        wh.plan(d, qs, k, aggs=[terms(0)], nested=[top(0)], window_collectors=False)
    assert e.value.rc == UNSUPPORTED and e.value.msg == "aggregations: more than 4 term clauses or top_k > 512 is not on the GPU path"


def test_narrow_flat_batch_is_the_flat_aggregation_plan(d):
    qs = [bq((0, S), (1, S)), bq((2, M), (RangeQuery(0, 0, 500_000), F)), bq((4, S), (5, S), (6, S), msm=2), MatchAllDocsQuery()]
    a = wh.plan(d, qs, 10, **COLLECTORS)
    b = wh.plan(d, qs, 10, window_collectors=False, **COLLECTORS)
    assert not a.wide and not a.tree and a.n_probe_simple + a.n_probe_generic == a.n_work > 0
    assert a.counters == b.counters
    assert a.clauses.tobytes() == b.clauses.tobytes() and a.queries.tobytes() == b.queries.tobytes()
    assert np.array_equal(a.work_query, b.work_query) and np.array_equal(a.work_item, b.work_item)
    assert bytes(a.aggs) == bytes(b.aggs) and bytes(a.nested) == bytes(b.nested)


def test_flat_batch_without_collectors_threshold_stays_exact(d):
    """the entry point forces exact collection: the request's threshold is INT32_MAX whatever the engine"""
    p = wh.plan(d, [bq((0, S), (1, S))], 10, aggs=[A(SUM, 0, 0, 0, 0, 0)])
    assert p.threshold == ph.INT_MAX


@pytest.mark.parametrize("case", ["terms", "metric", "nested"])
def test_multi_valued_column_is_unsupported(d, case):
    aggs = {"terms": [terms(1)], "metric": [A(MIN, 1, 0, 0, 0, 0)], "nested": [terms(0)]}[case]
    nested = [N(0, MAX, 1, 0, 0, 0, 0, 0)] if case == "nested" else []
    with pytest.raises(ph.PlanError) as e:
        wh.plan(d, TREES, 10, aggs=aggs, nested=nested)
    assert e.value.rc == UNSUPPORTED and "multi-valued column" in e.value.msg


def test_sort_on_a_tree_is_unsupported(d):
    with pytest.raises(ph.PlanError) as e:
        wh.plan(d, TREES, 10, aggs=[terms(0)], sort=_native.Sort(1, 0, 0, 0, 0, None))
    assert e.value.rc == UNSUPPORTED and e.value.msg == "sorted search of a query tree is not on the GPU path"


def test_more_than_8_aggregations_is_invalid(d):
    with pytest.raises(ph.PlanError) as e:
        wh.plan(d, TREES, 10, aggs=[A(SUM, 0, 0, 0, 0, 0)] * 9)
    assert e.value.rc == INVALID and e.value.msg == "at most 8 aggregations per search"


def test_filter_without_nested_collectors_is_invalid(d):
    with pytest.raises(ph.PlanError) as e:
        wh.plan(d, TREES, 10, aggs=[terms(0), A(FILTER, 0, 0, 0, 0, 0)], filters=[AggFilter(), AggFilter(1, 0, 0, 0, None)],
                filter_queries=[bq((8, S))])
    assert e.value.rc == INVALID and e.value.msg == 'Filter collector "aggs[1]" must have nested collectors'


def test_terms_table_limit_holds_on_trees(d):
    with pytest.raises(ph.PlanError) as e:
        wh.plan(d, TREES * 200, 10, aggs=[terms(2)])
    assert e.value.rc == UNSUPPORTED and "2 GB count table" in e.value.msg


def test_phrase_without_positions_keeps_its_refusal(d):
    with pytest.raises(ph.PlanError) as e:
        wh.plan(d, TREES, 10, aggs=[terms(0)], has_positions=False)
    assert e.value.rc == INVALID and "without position data" in e.value.msg
