"""ctypes binding of the test-only query-tree planner harness (tests/csrc/tree_plan_harness.cpp): the product's host
compiler and work planner (nrtsearch_b200/csrc/batch_plan.h, batch_plan.inc) run on a dictionary alone -- no postings, no
GPU -- for requests with nested queries (nrtgpu_search_tree), with the DevClause, DevQuery and DevNode records read back.
The dictionary and the errors are those of tests/plan_harness.py."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from nrtsearch_b200 import _native
from nrtsearch_b200.search import compile_tree
from plan_harness import CLAUSE, INT_MAX, QUERY, Dictionary, PlanError

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libtree_plan_harness.so")
NODE = np.dtype([("kind", "<i4"), ("clause_begin", "<i4"), ("n_clauses", "<i4"), ("n_req", "<i4"), ("need_should", "<i4"),
                 ("msm", "<i4"), ("tie_breaker", "<f4"), ("empty", "<i4")])
_COUNTERS = ("n_work", "n_probe_simple", "n_probe_generic", "parts_max", "n_lists", "n_slices", "slice_docs", "n_gran",
             "wide", "alg_postings", "threshold", "n_clauses", "tree", "n_nodes")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.th_last_error.restype = C.c_char_p
        h.th_plan.argtypes = [C.c_int32, C.c_int32, C.c_int32] + [C.c_void_p] * 5 + [C.c_int32, C.c_void_p, C.c_void_p] + \
                             [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p] + \
                             [C.c_int32] * 4 + [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
        h.th_free.argtypes = [C.c_void_p]
        h.th_counters.argtypes = [C.c_void_p, C.c_void_p]
        h.th_items.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        h.th_records.argtypes = [C.c_void_p] * 5
        assert (h.th_sizeof_clause(), h.th_sizeof_query(), h.th_sizeof_node()) == (CLAUSE.itemsize, QUERY.itemsize, NODE.itemsize)
        _lib = h
    return _lib


class TreePlan:
    """One compiled and planned request: counters (as tests/plan_harness.py's Plan, plus tree and n_nodes), the item
    list, the DevClause / DevQuery records and, for a tree batch, the DevNode records and each query's node range."""

    def __init__(self, handle: C.c_void_p, nq: int):
        h = lib()
        c = np.zeros(len(_COUNTERS), np.int64)
        h.th_counters(handle, c.ctypes.data)
        self.counters = dict(zip(_COUNTERS[:12], c[:12].tolist()))
        for k, v in zip(_COUNTERS, c.tolist()):
            setattr(self, k, v)
        self.wide, self.tree = bool(self.wide), bool(self.tree)
        self.work_query = np.zeros(self.n_work, np.int32)
        self.work_item = np.zeros(self.n_work, np.int32)
        h.th_items(handle, self.work_query.ctypes.data, self.work_item.ctypes.data)
        self.clauses = np.zeros(self.n_clauses, CLAUSE)
        self.queries = np.zeros(nq, QUERY)
        self.nodes = np.zeros(self.n_nodes, NODE)
        self.node_begin = np.zeros(nq + 1 if self.tree else 0, np.int32)
        h.th_records(handle, self.clauses.ctypes.data, self.queries.ctypes.data, self.nodes.ctypes.data, self.node_begin.ctypes.data)
        h.th_free(handle)

    def query_nodes(self, q):
        return self.nodes[self.node_begin[q]:self.node_begin[q + 1]]

    def query_clauses(self, q):
        qq = self.queries[q]
        return self.clauses[qq["clause_begin"]:qq["clause_begin"] + qq["n_clauses"]]


def plan_compiled(d: Dictionary, carr, ncl, narr, nn, qarr, nq, top_k: int, threshold: int = INT_MAX, sort=None, aggs=()):
    agg_arr = (_native.Aggregation * max(len(aggs), 1))(*aggs)
    h = C.c_void_p()
    rc = lib().th_plan(d.n_docs, d.doc_base, d.n_terms, d.term_off.ctypes.data, d.term_field.ctypes.data, d.term_df.ctypes.data,
                       d.term_max_x.ctypes.data, d.field_doc_count.ctypes.data, len(d.col_multi), d.col_multi.ctypes.data,
                       d.col_n_distinct.ctypes.data, int(d.has_deletes), 0, carr, ncl, narr, nn, qarr, nq, top_k, threshold, 0,
                       None if sort is None else C.byref(sort), agg_arr, len(aggs), C.byref(h))
    if rc != 0:
        raise PlanError(rc, lib().th_last_error().decode())
    return TreePlan(h, nq)


def plan(d: Dictionary, queries, top_k: int, threshold: int = INT_MAX, search_after=None, sort=None, aggs=()) -> TreePlan:
    """compile_batch (+ plan_work) of a tree request; raises PlanError with the product's status and message"""
    carr, ncl, narr, nn, qarr, nq = compile_tree(queries, search_after)
    return plan_compiled(d, carr, ncl, narr, nn, qarr, nq, top_k, threshold, sort, aggs)
