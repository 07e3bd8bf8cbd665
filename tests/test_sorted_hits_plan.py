"""The sorted-top-hits check of the host batch compiler (compile_batch), on the CPU through
tests/csrc/sorted_hits_plan_harness.cpp: an order on a record that is not TOP_HITS is NRTGPU_ERR_INVALID, orders_parent on a
sorted TOP_HITS keeps 'top hits cannot order the buckets', and the shapes of tests/test_filter_aggs_plan.py compile with
orders on their top hits. The refusals that need real orders (another index or leaf, leaf orders of different Sorts) are in
tests/test_gpu_sorted_hits.py. CPU only."""
import ctypes as C
import os

import numpy as np
import pytest

from filter_plan_harness import PlanError
from nrtsearch_b200 import _native
from nrtsearch_b200._native import AggFilter, Aggregation as A, NestedAggregation as N, NestedSort
from nrtsearch_b200.search import RangeQuery, compile_queries

INVALID = 1
TERMS, MIN, MAX, SUM, TOP_HITS, FILTER = 1, 2, 3, 4, 5, 6
ORDER = (C.c_void_p * 2)(0x1000, 0x2000)   # opaque to the compiler: any address stands for an order
SORTED, NONE = NestedSort(C.cast(ORDER, C.c_void_p), None), NestedSort()
_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libsorted_hits_plan_harness.so")


def lib():
    h = C.CDLL(_PATH)
    h.shp_last_error.restype = C.c_char_p
    h.shp_compile.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                              C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
    assert h.shp_sizeof_nested_sort() == C.sizeof(NestedSort)
    return h


def compile_sorted(aggs, nested, sorts, filters=None, filter_queries=(), col_multi=(0, 0, 0, 1), nq=4) -> int:
    """compile_batch with nested_sorts (None: no array); returns the nested records compiled with an order, raises PlanError"""
    cm = np.ascontiguousarray(col_multi, np.uint8)
    nd = np.full(len(cm), 10, np.int32)
    a = (_native.Aggregation * len(aggs))(*aggs)
    n = (_native.NestedAggregation * max(len(nested), 1))(*nested)
    s = None if sorts is None else (NestedSort * max(len(sorts), 1))(*sorts)
    f = None if filters is None else (AggFilter * len(filters))(*filters)
    carr, ncl, qarr, nfq = compile_queries(list(filter_queries)) if filter_queries else (None, 0, None, 0)
    out = C.c_int32(0)
    h = lib()
    rc = h.shp_compile(1000, len(cm), cm.ctypes.data, nd.ctypes.data, nq, a, len(aggs), n, len(nested), s, f, carr, ncl, qarr, nfq,
                       C.byref(out))
    if rc != 0:
        raise PlanError(rc, h.shp_last_error().decode())
    return out.value


def terms(col=0, filter_agg=0):
    return A(TERMS, col, 0, 10, 1, filter_agg)


def filt():
    return A(FILTER, 0, 0, 0, 0, 0)


def top(parent, hits=5, start=0, orders_parent=0):
    return N(parent, TOP_HITS, 0, 0, hits, start, orders_parent, 0)


def test_accepted_shapes():
    # sorted and relevance top hits under a terms aggregation, under a filter, and a filter's implicit match-all top level
    nested = [top(0, 7, 2), top(0, 4), N(0, MAX, 1, 0, 0, 0, 0, 0), top(1, 6), top(2, 3, 1)]
    qf = AggFilter(1, 0, 0, 0, None)
    assert compile_sorted([terms(), filt(), filt()], nested, [SORTED, NONE, NONE, SORTED, SORTED], [AggFilter(), qf, qf],
                          [RangeQuery(0, 0, 5)]) == 3
    assert compile_sorted([terms()], [top(0)], None) == 0                 # no array: every top hits by score
    assert compile_sorted([terms()], [top(0), N(0, MIN, 1, 0, 0, 0, 0, 0)], [NONE, NONE]) == 0


@pytest.mark.parametrize("kind", [MIN, MAX, SUM])
def test_order_on_a_metric_is_invalid(kind):
    with pytest.raises(PlanError) as e:
        compile_sorted([terms()], [top(0), N(0, kind, 1, 0, 0, 0, 0, 0)], [NONE, SORTED])
    assert e.value.rc == INVALID and e.value.msg == "nested aggregation: only top hits take a sort order"


def test_orders_parent_on_sorted_top_hits_keeps_its_refusal():
    with pytest.raises(PlanError) as e:
        compile_sorted([terms()], [top(0, orders_parent=1)], [SORTED])
    assert e.value.rc == INVALID and e.value.msg == "nested aggregation: top hits cannot order the buckets"
