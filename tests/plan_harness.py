"""ctypes binding of the test-only batch planner harness (tests/csrc/plan_harness.cpp): the product's host compiler and
probe work planner (nrtsearch_b200/csrc/batch_plan.h, batch_plan.inc) run on a dictionary alone -- no postings, no GPU.
The dictionary's tf planes and granule rows come from the index-build rules, and every work item is read back through
the decoder the probe kernel uses."""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Optional

import numpy as np

from nrtsearch_b200 import _native
from nrtsearch_b200.search import compile_queries

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libplan_harness.so")
_lib = None
INT_MAX = 2**31 - 1

CLAUSE = np.dtype([("post_base", "<i8"), ("n_post", "<i4"), ("occur", "<i4"), ("kind", "<i4"), ("slot", "<i4"),
                   ("field", "<i4"), ("col", "<i4"), ("weight", "<f4"), ("scoring", "<i4"), ("ub", "<f4"), ("plane", "<i4"),
                   ("gran_row", "<i4"), ("pad_", "<i4"), ("lo", "<i8"), ("hi", "<i8")])
QUERY = np.dtype([(n, "<i4") for n in ("clause_begin", "n_clauses", "n_term", "n_req", "need_should", "msm")] +
                 [(n, "<u4") for n in ("req_term_mask", "not_term_mask", "driver_mask")] +
                 [(n, "<i4") for n in ("dense_driver", "has_non_driver", "has_nonterm", "empty", "has_after")] +
                 [("must_term_mask", "<u4"), ("should_term_mask", "<u4"), ("nonterm_scoring", "<i4"), ("single_field", "<i4"),
                  ("after_key", "<u8")])
ITEM_WARM_DOCS, ITEM_BEHIND_WARM, ITEM_SWEEP = 1, 2, 4   # batch_plan.h kItem*
_COUNTERS = ("n_work", "n_probe_simple", "n_probe_generic", "parts_max", "n_lists", "n_slices", "slice_docs", "n_gran",
             "wide", "alg_postings", "threshold", "n_clauses")


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.ph_last_error.restype = C.c_char_p
        h.ph_bm25_cache.argtypes = [C.c_float, C.c_float, C.c_float, C.c_void_p]
        h.ph_index_rules.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        h.ph_plan.argtypes = [C.c_int32, C.c_int32, C.c_int32] + [C.c_void_p] * 5 + [C.c_int32, C.c_void_p, C.c_void_p] + \
                             [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p] + [C.c_int32] * 4 + \
                             [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]
        h.ph_free.argtypes = [C.c_void_p]
        for f in ("ph_counters", "ph_known_hits"):
            getattr(h, f).argtypes = [C.c_void_p, C.c_void_p]
        h.ph_items.argtypes = h.ph_records.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        h.ph_decode.argtypes = [C.c_int32, C.c_void_p]
        h.ph_span.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        h.ph_boundary_gran.argtypes = [C.c_void_p, C.c_int32]
        h.ph_boundary_gran.restype = C.c_int64
        assert h.ph_sizeof_clause() == CLAUSE.itemsize and h.ph_sizeof_query() == QUERY.itemsize
        _lib = h
    return _lib


def constants() -> dict:
    out = np.zeros(10, np.int64)
    lib().ph_constants(out.ctypes.data)
    keys = ("kT", "kGran", "kWarmGran", "kMaxSliceGran", "kWideSliceDocs", "kProbeMaxTopK", "kMaxTopK", "warm_min_docs",
            "slice_gran", "item_postings")
    return dict(zip(keys, out.tolist()))


def index_rules(n_docs: int, term_off) -> tuple[np.ndarray, np.ndarray]:
    """(term_plane, term_gran) of nrtgpu_index_build for a dictionary with these list offsets."""
    off = np.ascontiguousarray(term_off, np.int64)
    n = len(off) - 1
    tp, tg = np.empty(n, np.int32), np.empty(n, np.int32)
    lib().ph_index_rules(n_docs, n, off.ctypes.data, tp.ctypes.data, tg.ctypes.data)
    return tp, tg


def bm25_cache(k1: float, b: float, avgdl: float) -> np.ndarray:
    out = np.empty(256, np.float32)
    lib().ph_bm25_cache(k1, b, avgdl, out.ctypes.data)
    return out


def decode(w: int) -> tuple:
    """(slice, part, lparts, flags, sweep slot) of a work-item word."""
    out = np.empty(5, np.int32)
    lib().ph_decode(int(w), out.ctypes.data)
    return tuple(int(x) for x in out)


@dataclass
class Dictionary:
    """What the planner reads of a shard. term_max_x defaults to 1.0 per term, term_df to the list lengths,
    field_doc_count to n_docs."""
    n_docs: int
    term_off: np.ndarray
    term_field: Optional[np.ndarray] = None
    term_df: Optional[np.ndarray] = None
    term_max_x: Optional[np.ndarray] = None
    field_doc_count: Optional[np.ndarray] = None
    doc_base: int = 0
    col_multi: Optional[np.ndarray] = None
    col_n_distinct: Optional[np.ndarray] = None
    has_deletes: bool = False

    def __post_init__(self):
        self.term_off = np.ascontiguousarray(self.term_off, np.int64)
        n = len(self.term_off) - 1
        lens = np.diff(self.term_off)
        self.term_field = np.ascontiguousarray(np.zeros(n, np.int32) if self.term_field is None else self.term_field, np.int32)
        self.term_df = np.ascontiguousarray(lens if self.term_df is None else self.term_df, np.int64)
        self.term_max_x = np.ascontiguousarray(np.ones(n, np.float32) if self.term_max_x is None else self.term_max_x, np.float32)
        nf = int(self.term_field.max()) + 1 if n else 1
        self.field_doc_count = np.ascontiguousarray(np.full(nf, self.n_docs, np.int64) if self.field_doc_count is None
                                                    else self.field_doc_count, np.int64)
        self.col_multi = np.ascontiguousarray(np.zeros(0, np.uint8) if self.col_multi is None else self.col_multi, np.uint8)
        self.col_n_distinct = np.ascontiguousarray(np.zeros(len(self.col_multi), np.int32) if self.col_n_distinct is None
                                                   else self.col_n_distinct, np.int32)

    @property
    def n_terms(self) -> int:
        return len(self.term_off) - 1


class PlanError(Exception):
    def __init__(self, rc: int, msg: str):
        super().__init__(f"status {rc}: {msg}")
        self.rc, self.msg = rc, msg


class Plan:
    """One compiled (and planned) batch: counters, the item list, known hits and the DevClause / DevQuery records."""

    def __init__(self, handle: C.c_void_p, nq: int):
        h = lib()
        c = np.zeros(len(_COUNTERS), np.int64)
        h.ph_counters(handle, c.ctypes.data)
        self.counters = dict(zip(_COUNTERS, c.tolist()))
        for k, v in self.counters.items():
            setattr(self, k, v)
        self.wide = bool(self.wide)
        self.work_query = np.zeros(self.n_work, np.int32)
        self.work_item = np.zeros(self.n_work, np.int32)
        h.ph_items(handle, self.work_query.ctypes.data, self.work_item.ctypes.data)
        self.known_hits = np.zeros(nq, np.uint64)
        if self.n_slices:
            h.ph_known_hits(handle, self.known_hits.ctypes.data)
        self.clauses = np.zeros(self.n_clauses, CLAUSE)
        self.queries = np.zeros(nq, QUERY)
        h.ph_records(handle, self.clauses.ctypes.data, self.queries.ctypes.data)
        self._h = handle

    def span(self, w: int) -> tuple:
        """(g_lo, g_hi, e_lo, e_hi, out_list) of item w: what the probe kernel's item set-up computes."""
        out = np.empty(5, np.int32)
        lib().ph_span(self._h, int(w), out.ctypes.data)
        return tuple(int(x) for x in out)

    def boundary_gran(self, e: int) -> int:
        return int(lib().ph_boundary_gran(self._h, int(e)))

    def close(self):
        if self._h:
            lib().ph_free(self._h)
            self._h = None

    def __del__(self):
        self.close()


def plan(d: Dictionary, queries, top_k: int, threshold: int = INT_MAX, flags: int = 0, search_after=None, sort=None,
         aggs=(), sm_count: int = 0, do_plan: bool = True) -> Plan:
    """compile_batch (+ plan_work) of the product on dictionary d. Raises PlanError with the product's status and message."""
    carr, ncl, qarr, nq = compile_queries(queries, search_after)
    agg_arr = (_native.Aggregation * max(len(aggs), 1))(*aggs)
    h = C.c_void_p()
    rc = lib().ph_plan(d.n_docs, d.doc_base, d.n_terms, d.term_off.ctypes.data, d.term_field.ctypes.data, d.term_df.ctypes.data,
                       d.term_max_x.ctypes.data, d.field_doc_count.ctypes.data, len(d.col_multi), d.col_multi.ctypes.data,
                       d.col_n_distinct.ctypes.data, int(d.has_deletes), sm_count, carr, ncl, qarr, nq, top_k, threshold, flags,
                       None if sort is None else C.byref(sort), agg_arr, len(aggs), int(do_plan), C.byref(h))
    if rc != 0:
        raise PlanError(rc, lib().ph_last_error().decode())
    return Plan(h, nq)
