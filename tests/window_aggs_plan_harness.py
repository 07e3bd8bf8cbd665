"""ctypes binding of the test-only collector planner harness (tests/csrc/window_aggs_plan_harness.cpp): the product's host
compiler and work planner (nrtsearch_b200/csrc/batch_plan.h, batch_plan.inc) run on a dictionary alone -- no postings, no
GPU -- for the collector requests of nrtgpu_search_tree_aggs (query trees, phrases, wide batches), with window_collectors
set or not. The dictionary and the errors are those of tests/plan_harness.py."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from nrtsearch_b200 import _native
from nrtsearch_b200.search import compile_queries, compile_tree
from plan_harness import CLAUSE, QUERY, Dictionary, PlanError

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libwindow_aggs_plan_harness.so")
_COUNTERS = ("n_work", "n_probe_simple", "n_probe_generic", "n_lists", "n_slices", "slice_docs", "wide", "tree", "threshold",
             "n_clauses", "n_nodes", "n_phrases", "n_aggs", "n_nested", "n_sorted", "n_filters", "agg_filter_queries")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.wah_last_error.restype = C.c_char_p
        h.wah_plan.argtypes = [C.c_int32, C.c_int32] + [C.c_void_p] * 5 + [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32] + \
                              [C.c_void_p, C.c_int32] * 4 + [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32] + \
                              [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                               C.c_int32, C.POINTER(C.c_void_p)]
        h.wah_free.argtypes = [C.c_void_p]
        h.wah_counters.argtypes = [C.c_void_p, C.c_void_p]
        h.wah_collectors.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        h.wah_records.argtypes = [C.c_void_p] * 5
        assert (h.wah_sizeof_clause(), h.wah_sizeof_query()) == (CLAUSE.itemsize, QUERY.itemsize)
        _lib = h
    return _lib


class WindowAggsPlan:
    """One compiled and planned request: its counters as attributes, the compiled aggregation and nested records, the
    DevClause / DevQuery records and the item list."""

    def __init__(self, handle: C.c_void_p, nq: int):
        h = lib()
        c = np.zeros(len(_COUNTERS), np.int64)
        h.wah_counters(handle, c.ctypes.data)
        self.counters = dict(zip(_COUNTERS, c.tolist()))
        for k, v in self.counters.items():
            setattr(self, k, v)
        self.wide, self.tree = bool(self.wide), bool(self.tree)
        self.aggs = (_native.Aggregation * max(self.n_aggs, 1))()
        self.nested = (_native.NestedAggregation * max(self.n_nested, 1))()
        h.wah_collectors(handle, self.aggs, self.nested)
        self.clauses = np.zeros(self.n_clauses, CLAUSE)
        self.queries = np.zeros(nq, QUERY)
        self.work_query = np.zeros(self.n_work, np.int32)
        self.work_item = np.zeros(self.n_work, np.int32)
        h.wah_records(handle, self.clauses.ctypes.data, self.queries.ctypes.data, self.work_query.ctypes.data,
                      self.work_item.ctypes.data)
        h.wah_free(handle)


def plan(d: Dictionary, queries, top_k: int, aggs=(), nested=(), nested_sorts=None, filters=None, filter_queries=(), sort=None,
         window_collectors: bool = True, has_positions: bool = True) -> WindowAggsPlan:
    """compile_batch (+ plan_work) of the request nrtgpu_search_tree_aggs makes of these queries (compile_tree with the
    phrase table) and collectors; raises PlanError with the product's status and message"""
    carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(queries, phrase_table=True)
    a = (_native.Aggregation * max(len(aggs), 1))(*aggs)
    n = (_native.NestedAggregation * max(len(nested), 1))(*nested)
    s = None if nested_sorts is None else (_native.NestedSort * max(len(nested_sorts), 1))(*nested_sorts)
    f = None if filters is None else (_native.AggFilter * max(len(filters), 1))(*filters)
    fcarr, fncl, fqarr, fnq = compile_queries(list(filter_queries)) if filter_queries else (None, 0, None, 0)
    h = C.c_void_p()
    rc = lib().wah_plan(d.n_docs, d.n_terms, d.term_off.ctypes.data, d.term_field.ctypes.data, d.term_df.ctypes.data,
                        d.term_max_x.ctypes.data, d.field_doc_count.ctypes.data, len(d.col_multi), d.col_multi.ctypes.data,
                        d.col_n_distinct.ctypes.data, int(has_positions), carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, top_k,
                        None if sort is None else C.byref(sort), a, len(aggs), n, len(nested), s, f, fcarr, fncl, fqarr, fnq,
                        int(window_collectors), C.byref(h))
    if rc != 0:
        raise PlanError(rc, lib().wah_last_error().decode())
    return WindowAggsPlan(h, nq)
