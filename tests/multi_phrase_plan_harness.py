"""ctypes binding of the test-only multi-phrase planner harness (tests/csrc/multi_phrase_plan_harness.cpp): the product's
host compiler (nrtsearch_b200/csrc/batch_plan.inc compile_tree) on a dictionary alone -- no postings, no GPU -- for query
trees with multi-phrase leaves, with the DevClause, DevQuery and DevPhrase records and the batch's distinct unions read
back. The dictionary and the errors are those of tests/plan_harness.py."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from phrase_plan_harness import PHRASE
from plan_harness import CLAUSE, QUERY, Dictionary, PlanError  # noqa: F401  (Dictionary: the callers' argument)

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libmulti_phrase_plan_harness.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.mp_last_error.restype = C.c_char_p
        h.mp_plan.argtypes = [C.c_int32, C.c_int32] + [C.c_void_p] * 6 + [C.c_int64] + [C.c_void_p, C.c_int32] * 5 + \
                             [C.c_int32, C.POINTER(C.c_void_p)]
        h.mp_free.argtypes = [C.c_void_p]
        h.mp_counters.argtypes = [C.c_void_p, C.c_void_p]
        h.mp_records.argtypes = [C.c_void_p] * 10
        _lib = h
    return _lib


class MultiPhrasePlan:
    """One compiled request: clauses, queries, phrase records and ranges, and the unions (union_begin [n + 1], their
    terms, weights, modes -- 0 presence, 1 scored, 2 positions -- and the union clauses)"""

    def __init__(self, handle: C.c_void_p):
        h = lib()
        c = np.zeros(9, np.int64)
        h.mp_counters(handle, c.ctypes.data)
        n_cl, nq, _, n_ph, n_u, n_ut, n_uc, self.union_postings, self.union_positions = c.tolist()
        self.clauses, self.queries, self.phrases = np.zeros(n_cl, CLAUSE), np.zeros(nq, QUERY), np.zeros(n_ph, PHRASE)
        self.phrase_begin = np.zeros(nq + 1, np.int32)
        self.union_begin = np.zeros(n_u + 1 if n_u else 0, np.int32)
        self.union_term, self.union_weight = np.zeros(n_ut, np.int32), np.zeros(n_ut, np.float32)
        self.union_mode, self.union_clause = np.zeros(n_u, np.uint8), np.zeros(n_uc, np.int32)
        h.mp_records(handle, self.clauses.ctypes.data, self.queries.ctypes.data, self.phrases.ctypes.data,
                     self.phrase_begin.ctypes.data, self.union_begin.ctypes.data, self.union_term.ctypes.data,
                     self.union_weight.ctypes.data, self.union_mode.ctypes.data, self.union_clause.ctypes.data)
        h.mp_free(handle)

    def unions(self):
        return [self.union_term[self.union_begin[u]:self.union_begin[u + 1]].tolist() for u in range(len(self.union_mode))]

    def query_clauses(self, q):
        qq = self.queries[q]
        return self.clauses[qq["clause_begin"]:qq["clause_begin"] + qq["n_clauses"]]


def plan_compiled(d, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, top_k: int = 10, term_pos=None,
                  max_union_postings: int = 0) -> MultiPhrasePlan:
    """compile_batch of compile_tree(..., phrase_table=True)'s arrays with multi-phrases accepted; term_pos: [n_terms + 1]
    first position of each term (None: no positions); raises PlanError with the product's status and message"""
    h = C.c_void_p()
    tp = None if term_pos is None else np.ascontiguousarray(term_pos, np.int64)
    rc = lib().mp_plan(d.n_docs, d.n_terms, d.term_off.ctypes.data, d.term_field.ctypes.data, d.term_df.ctypes.data,
                       d.term_max_x.ctypes.data, d.field_doc_count.ctypes.data, None if tp is None else tp.ctypes.data,
                       max_union_postings, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, top_k, C.byref(h))
    if rc != 0:
        raise PlanError(rc, lib().mp_last_error().decode())
    return MultiPhrasePlan(h)
