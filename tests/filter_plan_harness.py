"""ctypes binding of the test-only filter-collector harness (tests/csrc/filter_plan_harness.cpp): the product's host compiler
(compile_batch, nrtsearch_b200/csrc/batch_plan.inc) on one request with aggregations, nested collectors and filter records,
on a dictionary of columns alone -- no postings, no GPU."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from nrtsearch_b200 import _native
from nrtsearch_b200.search import compile_queries

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libfilter_plan_harness.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.fph_last_error.restype = C.c_char_p
        h.fph_compile.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                  C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
        assert h.fph_sizeof_agg_filter() == C.sizeof(_native.AggFilter)
        _lib = h
    return _lib


class PlanError(Exception):
    def __init__(self, rc: int, msg: str):
        super().__init__(f"status {rc}: {msg}")
        self.rc, self.msg = rc, msg


def compile_aggs(aggs, nested=(), filters=None, filter_queries=(), n_docs=1000, col_multi=(0, 0, 0, 1), n_distinct=None,
                 nq=4) -> int:
    """compile_batch of nq match-all queries with these records (filters: one nrtgpu_agg_filter per aggregation, or None
    for no array); returns the aggregations compiled, raises PlanError with the product's status and message"""
    cm = np.ascontiguousarray(col_multi, np.uint8)
    nd = np.ascontiguousarray(n_distinct if n_distinct is not None else [10] * len(cm), np.int32)
    a = (_native.Aggregation * max(len(aggs), 1))(*aggs)
    n = (_native.NestedAggregation * max(len(nested), 1))(*nested)
    f = None if filters is None else (_native.AggFilter * max(len(filters), 1))(*filters)
    carr, ncl, qarr, nfq = compile_queries(list(filter_queries)) if filter_queries else (None, 0, None, 0)
    out = C.c_int32(0)
    rc = lib().fph_compile(n_docs, len(cm), cm.ctypes.data, nd.ctypes.data, nq, a, len(aggs), n, len(nested), f, carr, ncl, qarr,
                           nfq, C.byref(out))
    if rc != 0:
        raise PlanError(rc, lib().fph_last_error().decode())
    return out.value
