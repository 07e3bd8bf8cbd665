"""ctypes binding of the test-only block-join planner harness (tests/csrc/nested_plan_harness.cpp): the product's host
compiler and work planner (nrtsearch_b200/csrc/batch_plan.inc compile_tree / plan_work) on a dictionary alone -- no
postings, no GPU -- for query trees with NestedQuery nodes, with the DevClause, DevQuery and DevNode records, the joins
and the two passes' work items read back. The dictionary and the errors are those of tests/plan_harness.py."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from plan_harness import CLAUSE, QUERY, Dictionary, PlanError  # noqa: F401  (Dictionary: the callers' argument)
from tree_plan_harness import NODE

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libnested_plan_harness.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.nj_last_error.restype = C.c_char_p
        h.nj_plan.argtypes = [C.c_int32, C.c_int32] + [C.c_void_p] * 5 + [C.c_int64, C.c_int64] + [C.c_void_p, C.c_int32] * 5 + \
                             [C.c_int32, C.POINTER(C.c_void_p)]
        h.nj_free.argtypes = [C.c_void_p]
        h.nj_counters.argtypes = [C.c_void_p, C.c_void_p]
        h.nj_records.argtypes = [C.c_void_p] * 9
        _lib = h
    return _lib


class NestedPlan:
    """One compiled and planned request: clauses, queries (the request's, then one child query per join), nodes and their
    per-query ranges, the joins (clause, mode), their bound, and the query of every parent-pass and child-pass item"""

    def __init__(self, handle: C.c_void_p):
        h = lib()
        c = np.zeros(8, np.int64)
        h.nj_counters(handle, c.ctypes.data)
        n_cl, n_q, n_nodes, n_joins, self.join_bound, n_work, n_jwork, self.n_slices = c.tolist()
        self.clauses, self.queries, self.nodes = np.zeros(n_cl, CLAUSE), np.zeros(n_q, QUERY), np.zeros(n_nodes, NODE)
        self.node_begin = np.zeros(n_q + 1, np.int32)
        self.join_clause, self.join_mode = np.zeros(n_joins, np.int32), np.zeros(n_joins, np.uint8)
        self.work_query, self.join_query = np.zeros(n_work, np.int32), np.zeros(n_jwork, np.int32)
        h.nj_records(handle, self.clauses.ctypes.data, self.queries.ctypes.data, self.nodes.ctypes.data, self.node_begin.ctypes.data,
                     self.join_clause.ctypes.data, self.join_mode.ctypes.data, self.work_query.ctypes.data,
                     self.join_query.ctypes.data)
        h.nj_free(handle)

    def query_clauses(self, q):
        qq = self.queries[q]
        return self.clauses[qq["clause_begin"]:qq["clause_begin"] + qq["n_clauses"]]

    def query_nodes(self, q):
        return self.nodes[self.node_begin[q]:self.node_begin[q + 1]]


def plan_compiled(d, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, top_k: int = 10, n_parents: int = 1000,
                  max_join_children: int = 0) -> NestedPlan:
    """compile_batch + plan_work of compile_tree(..., phrase_table=True)'s arrays with joins accepted; n_parents < 0: an
    image without parents; raises PlanError with the product's status and message"""
    h = C.c_void_p()
    rc = lib().nj_plan(d.n_docs, d.n_terms, d.term_off.ctypes.data, d.term_field.ctypes.data, d.term_df.ctypes.data,
                       d.term_max_x.ctypes.data, d.field_doc_count.ctypes.data, n_parents, max_join_children, carr, ncl, narr, nn,
                       parr, n_ph, tarr, n_pt, qarr, nq, top_k, C.byref(h))
    if rc != 0:
        raise PlanError(rc, lib().nj_last_error().decode())
    return NestedPlan(h)
