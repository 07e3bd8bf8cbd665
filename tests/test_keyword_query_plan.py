"""Keyword range clauses (NRTGPU_KEYWORD_RANGE) in the host batch compiler, through the test-only harness
tests/csrc/keyword_query_harness.cpp (batch_plan.inc on a dictionary alone, no GPU): validation and its messages, the
driver a query gets, trees, and keyword value sets of filter collectors."""
import ctypes as C
import os

import numpy as np
import pytest

from nrtsearch_b200._native import AggFilter as F, Clause, Node, Query

OK, INVALID = 0, 1
SHOULD, MUST, FILTER, MUST_NOT = 0, 1, 2, 3
TERM, RANGE, MATCH_ALL, NODE, KEYWORD = 0, 1, 2, 3, 5
_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libkeyword_query_harness.so")
# three terms of 5000, 300 and 40000 postings on a 100K-doc shard; two numeric columns; keyword columns of 500 and 3 terms
N_DOCS = 100_000
TERM_OFF = np.array([0, 5000, 5300, 45300], np.int64)
KW_TERMS = np.array([500, 3], np.int32)


@pytest.fixture(scope="module")
def lib():
    h = C.CDLL(_PATH)
    h.kqh_last_error.restype = C.c_char_p
    h.kqh_compile.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                              C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
    h.kqh_compile_filters.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32]
    return h


def compile_(lib, queries, nodes=(), kw_terms=KW_TERMS, top_k=10):
    """queries: lists of (occur, kind, id, boost, lo, hi) clause tuples (the root's); nodes: (kind, begin, end, msm, tie, 0)
    over the clause array after the roots' clauses. Returns (status, message, dense, driver, nonterm)."""
    flat, qs = [], []
    for cls in queries:
        qs.append((len(flat), len(flat) + len(cls), 0, 0, 0, 0.0))
        flat += cls
    base = len(flat)
    nd = []
    for kind, b, e, msm, tie, extra in nodes:
        nd.append((kind, base + b, base + e, msm, tie, 0))
        flat += extra
    carr = (Clause * max(len(flat), 1))(*[Clause(*c) for c in flat])
    qarr = (Query * len(qs))(*[Query(*q) for q in qs])
    narr = (Node * max(len(nd), 1))(*[Node(*n) for n in nd]) if nd else None
    nq = len(qs)
    dense, driver, nonterm = np.zeros(nq, np.int32), np.zeros(nq, np.uint32), np.zeros(nq, np.int32)
    rc = lib.kqh_compile(N_DOCS, len(TERM_OFF) - 1, TERM_OFF.ctypes.data, 2, len(kw_terms), kw_terms.ctypes.data, carr, len(flat),
                         qarr, nq, narr, len(nd), top_k, dense.ctypes.data, driver.ctypes.data, nonterm.ctypes.data)
    return rc, lib.kqh_last_error().decode(), dense, driver, nonterm


def kw(occur, column=0, lo=1, hi=1001, boost=1.0):
    return (occur, KEYWORD, column, boost, lo, hi)


@pytest.mark.parametrize("occur", [SHOULD, MUST, FILTER])
def test_keyword_only_queries_take_the_dense_driver(lib, occur):
    rc, _, dense, _, nonterm = compile_(lib, [[kw(occur, 0, 10, 20)], [kw(occur, 1, 1, 7), kw(SHOULD, 0, 3, 3)]])
    assert rc == OK and dense.tolist() == [1, 1]
    scoring = occur != FILTER
    assert nonterm[0] == (1 | (2 if scoring else 0))


def test_the_rarest_required_term_still_leads(lib):
    rc, _, dense, driver, _ = compile_(lib, [[(MUST, TERM, 2, 1.0, 0, 0), kw(FILTER), (MUST, TERM, 1, 1.0, 0, 0)],
                                             [(SHOULD, TERM, 0, 1.0, 0, 0), (SHOULD, TERM, 1, 1.0, 0, 0), kw(MUST_NOT)],
                                             [(SHOULD, TERM, 0, 1.0, 0, 0), kw(SHOULD)]])
    assert rc == OK
    assert dense.tolist() == [0, 0, 1]
    assert driver[0] == 1 << 1        # term 1 (300 postings) is slot 1 and leads
    assert driver[1] == 0b11          # a MUST_NOT keyword clause leaves a pure disjunction's drivers alone


def test_empty_range_is_accepted(lib):
    assert compile_(lib, [[kw(MUST, 0, 9, 4)], [kw(FILTER, 1, 7, 1)]])[0] == OK


@pytest.mark.parametrize("column", [-1, 2])
def test_keyword_column_out_of_range(lib, column):
    rc, msg, *_ = compile_(lib, [[kw(MUST, column, 1, 1)]])
    assert rc == INVALID and "keyword column out of range" in msg


def test_image_without_keyword_columns(lib):
    rc, msg, *_ = compile_(lib, [[kw(MUST, 0, 1, 1)]], kw_terms=np.zeros(0, np.int32))
    assert rc == INVALID and "keyword column out of range" in msg


@pytest.mark.parametrize("lo,hi", [(0, 5), (5, 0), (1, 1002), (1002, 3), (-4, 4)])
def test_keyword_code_out_of_range(lib, lo, hi):
    rc, msg, *_ = compile_(lib, [[kw(MUST, 0, lo, hi)]])
    assert rc == INVALID and "keyword code out of range" in msg


def test_code_bounds_are_per_column(lib):
    assert compile_(lib, [[kw(MUST, 1, 1, 7)]])[0] == OK
    assert compile_(lib, [[kw(MUST, 1, 1, 8)]])[1].endswith("keyword code out of range")


def test_trees_accept_the_clause(lib):
    # root: MUST node(BOOL: SHOULD term 0, SHOULD keyword), FILTER keyword; the node's keyword clause is checked too
    node = [(0, 0, 2, 0, 0.0, [(SHOULD, TERM, 0, 1.0, 0, 0), kw(SHOULD, 0, 2, 40)])]
    rc, _, dense, _, _ = compile_(lib, [[(MUST, NODE, 0, 1.0, 0, 0), kw(FILTER, 1, 2, 2)]], node)
    assert rc == OK and dense.tolist() == [1]   # a SHOULD keyword clause leaves the node without a cover
    bad = [(0, 0, 1, 0, 0.0, [kw(MUST, 0, 2, 1002)])]
    rc, msg, *_ = compile_(lib, [[(MUST, NODE, 0, 1.0, 0, 0)]], bad)
    assert rc == INVALID and "keyword code out of range" in msg


def test_kind_7_is_still_a_bad_clause_kind(lib):
    rc, msg, *_ = compile_(lib, [[(MUST, 7, 0, 1.0, 0, 0)]])
    assert rc == INVALID and msg == "bad clause kind"


def compile_filters(lib, filters, kw_terms=KW_TERMS):
    keep = [np.asarray(v, np.int64) for _, _, v in filters]
    arr = (F * len(filters))(*[F(kind, 0, col, len(v), v.ctypes.data if len(v) else None) for (kind, col, _), v in zip(filters, keep)])
    rc = lib.kqh_compile_filters(len(kw_terms), kw_terms.ctypes.data, arr, len(filters))
    return rc, lib.kqh_last_error().decode()


def test_keyword_value_sets(lib):
    KWSET = 4   # NRTGPU_AGG_FILTER_KEYWORD_SET (3 stays a bad filter kind)
    assert compile_filters(lib, [(KWSET, 0, [2, 3, 1001]), (KWSET, 1, [])])[0] == OK
    assert compile_filters(lib, [(KWSET, 2, [2])]) == (INVALID, "filter aggregation: keyword column out of range")
    assert compile_filters(lib, [(KWSET, 1, [0])]) == (INVALID, "filter aggregation: keyword code out of range")
    assert compile_filters(lib, [(KWSET, 1, [8])]) == (INVALID, "filter aggregation: keyword code out of range")
    assert compile_filters(lib, [(3, 0, [2])]) == (INVALID, "filter aggregation: bad filter kind")
    assert compile_filters(lib, [(5, 0, [2])]) == (INVALID, "filter aggregation: bad filter kind")
