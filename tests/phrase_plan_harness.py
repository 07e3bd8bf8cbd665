"""ctypes binding of the test-only phrase planner harness (tests/csrc/phrase_plan_harness.cpp): the product's host compiler
and work planner (nrtsearch_b200/csrc/batch_plan.h, batch_plan.inc) run on a dictionary alone -- no postings, no GPU -- for
query trees with phrase leaves (nrtgpu_search_tree_phrases), with the DevClause, DevQuery, DevNode and DevPhrase records read
back. The dictionary and the errors are those of tests/plan_harness.py."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from plan_harness import CLAUSE, INT_MAX, QUERY, Dictionary, PlanError
from tree_plan_harness import NODE

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libphrase_plan_harness.so")
PHRASE = np.dtype([("clause0", "<i4"), ("n_terms", "<i4"), ("slop", "<i4"), ("field", "<i4"), ("weight", "<f4"),
                   ("cover_slot", "<i4"), ("reserved", "<i4", 2), ("offset", "<i4", 8)])
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.pp_last_error.restype = C.c_char_p
        h.pp_plan.argtypes = [C.c_int32, C.c_int32] + [C.c_void_p] * 5 + [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p] + \
                             [C.c_void_p, C.c_int32] * 4 + [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
        h.pp_free.argtypes = [C.c_void_p]
        h.pp_counters.argtypes = [C.c_void_p, C.c_void_p]
        h.pp_records.argtypes = [C.c_void_p] * 7
        assert (h.pp_sizeof_clause(), h.pp_sizeof_query(), h.pp_sizeof_node(), h.pp_sizeof_phrase()) == \
            (CLAUSE.itemsize, QUERY.itemsize, NODE.itemsize, PHRASE.itemsize)
        _lib = h
    return _lib


class PhrasePlan:
    """One compiled request: the DevClause / DevQuery / DevNode / DevPhrase records, each query's node and phrase ranges,
    alg_postings and the work items planned."""

    def __init__(self, handle: C.c_void_p):
        h = lib()
        c = np.zeros(7, np.int64)
        h.pp_counters(handle, c.ctypes.data)
        n_cl, nq, n_nodes, n_ph, tree, self.alg_postings, self.n_work = c.tolist()
        self.tree = bool(tree)
        self.clauses, self.queries = np.zeros(n_cl, CLAUSE), np.zeros(nq, QUERY)
        self.nodes, self.phrases = np.zeros(n_nodes, NODE), np.zeros(n_ph, PHRASE)
        self.node_begin = np.zeros(nq + 1 if tree else 0, np.int32)
        self.phrase_begin = np.zeros(nq + 1 if tree else 0, np.int32)
        h.pp_records(handle, self.clauses.ctypes.data, self.queries.ctypes.data, self.nodes.ctypes.data, self.node_begin.ctypes.data,
                     self.phrases.ctypes.data, self.phrase_begin.ctypes.data)
        h.pp_free(handle)

    def query_clauses(self, q):
        qq = self.queries[q]
        return self.clauses[qq["clause_begin"]:qq["clause_begin"] + qq["n_clauses"]]


def plan_compiled(d: Dictionary, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, top_k: int = 10,
                  threshold: int = INT_MAX, positions: bool = True) -> PhrasePlan:
    """compile_batch (+ plan_work) of compile_tree(..., phrase_table=True)'s arrays on an image with or without positions;
    raises PlanError with the product's status and message"""
    h = C.c_void_p()
    rc = lib().pp_plan(d.n_docs, d.n_terms, d.term_off.ctypes.data, d.term_field.ctypes.data, d.term_df.ctypes.data,
                       d.term_max_x.ctypes.data, d.field_doc_count.ctypes.data, int(positions), len(d.col_multi),
                       d.col_multi.ctypes.data, d.col_n_distinct.ctypes.data, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq,
                       top_k, threshold, C.byref(h))
    if rc != 0:
        raise PlanError(rc, lib().pp_last_error().decode())
    return PhrasePlan(h)
