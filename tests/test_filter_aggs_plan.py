"""The filter-collector checks of the host batch compiler (compile_batch), on the CPU through tests/filter_plan_harness.py:
every INVALID rule of nrtgpu_search_bool_aggs_filtered with its message, and the shapes it accepts. CPU only."""
import ctypes as C

import pytest

from filter_plan_harness import PlanError, compile_aggs, lib
from nrtsearch_b200 import _native
from nrtsearch_b200._native import AggFilter, Aggregation as A, NestedAggregation as N
from nrtsearch_b200.search import RangeQuery

INVALID, UNSUPPORTED = 1, 3
TERMS, MIN, MAX, SUM, TOP_HITS, FILTER = 1, 2, 3, 4, 5, 6
QUERY, VALUE_SET = 1, 2
NONE = AggFilter()


def terms(col=0, filter_agg=0):
    return A(TERMS, col, 0, 10, 1, filter_agg)


def filt(filter_agg=0):
    return A(FILTER, 0, 0, 0, 0, filter_agg)


def qf(i=0):
    return AggFilter(QUERY, i, 0, 0, None)


def vs(col=1, n=0):
    return AggFilter(VALUE_SET, 0, col, n, None)


RANGE = RangeQuery(0, 0, 5)


def test_accepted_shapes():
    # a terms collector under a query filter; a filter under it with a value set; nested metrics and top hits under both
    aggs = [filt(), terms(0, 1), filt(1), terms(2, 3)]
    nested = [N(0, MAX, 0, 0, 0, 0, 0, 0), N(2, TOP_HITS, 0, 0, 5, 0, 0, 0), N(1, SUM, 2, 0, 0, 0, 0, 0)]
    assert compile_aggs(aggs, nested, [qf(), NONE, vs(3), NONE], [RANGE]) == 4
    # a value set on a multi-valued column (3), an empty set; a filter with only nested collectors
    assert compile_aggs([filt()], [N(0, MIN, 0, 0, 0, 0, 0, 0)], [vs(3, 0)]) == 1
    # existing shapes keep compiling without filter records
    assert compile_aggs([terms(), A(MAX, 1, 0, 0, 0, 0)], [N(0, TOP_HITS, 0, 0, 3, 1, 0, 0)]) == 2


@pytest.mark.parametrize("aggs, nested, filters, fq, rc, msg", [
    ([filt()], [], [qf()], [RANGE], INVALID, 'Filter collector "aggs[0]" must have nested collectors'),
    ([filt(), filt(1)], [], [qf(), qf()], [RANGE], INVALID, 'Filter collector "aggs[1]" must have nested collectors'),
    ([filt(), terms()], [], None, [], INVALID, "filter aggregation: no filter records"),
    ([filt(), terms(0, 1)], [], [AggFilter(3, 0, 0, 0, None), NONE], [], INVALID, "filter aggregation: bad filter kind"),
    ([filt(), terms(0, 1)], [], [AggFilter(0, 0, 0, 0, None), NONE], [], INVALID, "filter aggregation: bad filter kind"),
    ([filt(), terms(0, 1)], [], [qf(1), NONE], [RANGE], INVALID, "filter aggregation: filter query out of range"),
    ([filt(), terms(0, 1)], [], [qf(-1), NONE], [RANGE], INVALID, "filter aggregation: filter query out of range"),
    ([filt(), terms(0, 1)], [], [qf(0), NONE], [], INVALID, "filter aggregation: filter query out of range"),
    ([filt(), terms(0, 1)], [], [vs(4), NONE], [], INVALID, "filter aggregation: column out of range"),
    ([filt(), terms(0, 1)], [], [vs(-1), NONE], [], INVALID, "filter aggregation: column out of range"),
    ([filt(), terms(0, 1)], [], [vs(1, -1), NONE], [], INVALID, "filter aggregation: bad value set"),
    ([filt(), terms(0, 1)], [], [vs(1, 2), NONE], [], INVALID, "filter aggregation: bad value set"),   # values NULL
    ([filt(), A(MAX, 0, 0, 0, 0, 1)], [], [qf(), NONE], [RANGE], INVALID,
     "filter aggregation: only terms and filter aggregations take filter_agg"),
    ([filt(), terms(0, 2)], [], [qf(), NONE], [RANGE], INVALID, "filter aggregation: filter_agg must name an earlier filter aggregation"),
    ([terms(0, 2), filt()], [], [NONE, qf()], [RANGE], INVALID, "filter aggregation: filter_agg must name an earlier filter aggregation"),
    ([filt(), terms(0, 1), terms(0, 2)], [], [qf(), NONE, NONE], [RANGE], INVALID,
     "filter aggregation: filter_agg must name an earlier filter aggregation"),   # names a terms aggregation
    ([filt(), terms(0, -1)], [], [qf(), NONE], [RANGE], INVALID, "filter aggregation: filter_agg must name an earlier filter aggregation"),
    ([filt(1)], [N(0, MAX, 0, 0, 0, 0, 0, 0)], [qf()], [RANGE], INVALID, "filter aggregation: filter_agg must name an earlier filter aggregation"),
    ([filt()], [N(0, MAX, 0, 0, 0, 0, 1, 0)], [qf()], [RANGE], INVALID, "nested aggregation: a filter aggregation has no buckets to order"),
    ([filt()], [N(0, FILTER, 0, 0, 0, 0, 0, 0)], [qf()], [RANGE], INVALID, "bad nested aggregation kind"),
    ([filt()], [N(0, MAX, 3, 0, 0, 0, 0, 0)], [qf()], [RANGE], UNSUPPORTED, "nested aggregation on a multi-valued column"),
    ([filt()] * 5, [N(0, MAX, 0, 0, 0, 0, 0, 0)] * 5, [qf()] * 5, [RANGE], UNSUPPORTED,
     "more than 4 nested aggregations on one terms aggregation"),
    ([filt()] + [terms(0, 1)] * 8, [], [qf()] + [NONE] * 8, [RANGE], INVALID, "at most 8 aggregations per search"),
    ([filt(), terms(3, 1)], [], [qf(), NONE], [RANGE], UNSUPPORTED, "aggregation on a multi-valued column"),
    ([A(0, 0, 0, 0, 0, 0)], [], [NONE], [], INVALID, "bad aggregation kind"),
    ([A(TOP_HITS, 0, 0, 0, 0, 0)], [], [NONE], [], INVALID, "bad aggregation kind"),
    ([A(7, 0, 0, 0, 0, 0)], [], [NONE], [], INVALID, "bad aggregation kind"),
])
def test_refusals(aggs, nested, filters, fq, rc, msg):
    with pytest.raises(PlanError) as e:
        compile_aggs(aggs, nested, filters, fq)
    assert (e.value.rc, e.value.msg) == (rc, msg)


def test_filter_query_with_search_after_is_refused():
    carr = (_native.Clause * 1)(_native.Clause(1, 2, 0, 1.0, 0, 0))
    qarr = (_native.Query * 1)(_native.Query(0, 1, 0, 1, 3, 1.0))
    aggs = (_native.Aggregation * 2)(filt(), terms(0, 1))
    f = (_native.AggFilter * 2)(qf(), NONE)
    cm = (C.c_uint8 * 4)(0, 0, 0, 1)
    nd = (C.c_int32 * 4)(10, 10, 10, 10)
    out = C.c_int32()
    assert lib().fph_compile(100, 4, cm, nd, 2, aggs, 2, None, 0, f, carr, 1, qarr, 1, C.byref(out)) == INVALID
    assert lib().fph_last_error().decode() == "filter aggregation: a filter query has no searchAfter"


def test_nested_top_hits_under_a_filter_count_one_bucket():
    # nq * size * top_hits: a filter's size is 1, so 2^24 / 1024 queries of top 1024 fit and one more query does not
    n = N(0, TOP_HITS, 0, 0, 1024, 0, 0, 0)
    assert compile_aggs([filt()], [n], [vs(1)], nq=16384) == 1
    with pytest.raises(PlanError) as e:
        compile_aggs([filt()], [n], [vs(1)], nq=16385)
    assert e.value.rc == UNSUPPORTED

