"""The keyword-terms rules of the host batch compiler and the checks of nrtgpu_index_add_keyword_columns, through the
test-only planner harness tests/csrc/keyword_plan_harness.cpp (batch_plan.inc on a dictionary alone, no GPU)."""
import ctypes as C
import os

import numpy as np
import pytest

from nrtsearch_b200._native import Aggregation as A, KeywordColumn as KC, NestedAggregation as N

OK, INVALID, UNSUPPORTED = 0, 1, 3
TERMS, MIN, MAX, SUM, TOP_HITS = 1, 2, 3, 4, 5
KW = 3
_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libkeyword_plan_harness.so")


@pytest.fixture(scope="module")
def lib():
    h = C.CDLL(_PATH)
    h.kph_last_error.restype = C.c_char_p
    h.kph_compile.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                              C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
    h.kph_check_keyword_columns.argtypes = [C.c_int32, C.c_void_p, C.c_int32]
    assert h.kph_sizeof_keyword_column() == C.sizeof(KC)
    return h


# two numeric columns (one multi-valued), keyword columns: 0 SORTED of 500 terms, 1 SORTED_SET of 300 terms, 2 of 3 terms
MULTI = np.array([0, 1], np.uint8)
DISTINCT = np.array([100, 0], np.int32)
KW_TERMS = np.array([500, 300, 3], np.int32)


def compile_aggs(lib, aggs, nested=(), nq=4, kw_terms=KW_TERMS):
    a = (A * len(aggs))(*aggs)
    n = (N * max(len(nested), 1))(*nested)
    out = C.c_int32(-1)
    rc = lib.kph_compile(1000, 2, MULTI.ctypes.data, DISTINCT.ctypes.data, 3, kw_terms.ctypes.data, nq,
                         a, len(aggs), n if nested else None, len(nested), C.byref(out))
    return rc, lib.kph_last_error().decode(), out.value


def test_keyword_terms_accepted(lib):
    assert compile_aggs(lib, [A(TERMS, 0, KW, 10, 1, 0)])[0] == OK
    assert compile_aggs(lib, [A(TERMS, 1, KW, 2048, 0, 0), A(TERMS, 0, 0, 5, 1, 0)],
                        [N(0, MAX, 0, 0, 0, 0, 1, 0), N(0, TOP_HITS, 0, 0, 3, 0, 0, 0)])[::2] == (OK, 2)
    eight = [A(TERMS, k % 3, KW, 5, k % 2, 0) for k in range(8)]   # keyword terms take one collector slot each, as numeric ones do
    assert compile_aggs(lib, eight)[::2] == (OK, 8)
    assert compile_aggs(lib, eight + [A(TERMS, 0, KW, 5, 1, 0)])[:2] == (INVALID, "at most 8 aggregations per search")


@pytest.mark.parametrize("kind", [MIN, MAX, SUM])
def test_metrics_on_a_keyword_column_refused(lib, kind):
    assert compile_aggs(lib, [A(kind, 0, KW, 0, 0, 0)])[:2] == (INVALID, "bad aggregation value_type")


@pytest.mark.parametrize("col", [-1, 3])
def test_keyword_column_out_of_range(lib, col):
    assert compile_aggs(lib, [A(TERMS, col, KW, 10, 1, 0)])[:2] == (INVALID, "terms aggregation: keyword column out of range")


def test_nested_keyword_value_type_refused(lib):
    assert compile_aggs(lib, [A(TERMS, 0, KW, 10, 1, 0)], [N(0, MIN, 0, KW, 0, 0, 0, 0)])[:2] == \
        (INVALID, "bad nested aggregation value_type")


def test_size_and_table_limits(lib):
    for size in (0, 2049):
        assert compile_aggs(lib, [A(TERMS, 0, KW, size, 1, 0)])[:2] == (UNSUPPORTED, "terms aggregation: size must be in [1, 2048]")
    big = np.array([1 << 20, 300, 3], np.int32)
    assert compile_aggs(lib, [A(TERMS, 0, KW, 10, 1, 0)], nq=512, kw_terms=big)[0] == OK          # 2^29 cells: 2 GB exactly
    assert compile_aggs(lib, [A(TERMS, 0, KW, 10, 1, 0)], nq=513, kw_terms=big)[:2] == \
        (UNSUPPORTED, "terms aggregation: batch x distinct values exceeds the 2 GB count table")
    assert compile_aggs(lib, [A(TERMS, 0, KW, 10, 1, 0)], [N(0, SUM, 0, 0, 0, 0, 0, 0)], nq=257, kw_terms=big)[:2] == \
        (UNSUPPORTED, "nested aggregation: batch x distinct values exceeds the 2 GB table")


def column(terms, ords, offsets=None):
    keep = []
    tb = np.frombuffer(b"".join(terms) or b"\0", np.uint8).copy()
    toff = np.zeros(len(terms) + 1, np.int64)
    np.cumsum([len(t) for t in terms], out=toff[1:])
    o = np.asarray(ords, np.int32)
    off = None if offsets is None else np.asarray(offsets, np.int64)
    keep += [tb, toff, o, off]
    c = KC(len(terms), 0 if off is None else 1, tb.ctypes.data, toff.ctypes.data, o.ctypes.data if len(o) else None,
           None if off is None else off.ctypes.data)
    return c, keep


def check(lib, n_docs, *cols):
    arr = (KC * len(cols))(*[c for c, _ in cols])
    rc = lib.kph_check_keyword_columns(n_docs, arr, len(cols))
    return rc, lib.kph_last_error().decode()


def test_valid_columns(lib):
    assert check(lib, 3, column([b"a", b"b"], [0, -1, 1]), column([b"", b"a", b"ab", b"b"], [0, 2, 1, 3], [0, 2, 2, 4]))[0] == OK
    assert check(lib, 2, column([], [-1, -1]))[0] == OK


@pytest.mark.parametrize("terms,ords,offsets,msg", [
    ([b"b", b"a"], [0, 1], None, "column 0: terms must be strictly ascending in byte order (term 1)"),
    ([b"a", b"a"], [0, 1], None, "column 0: terms must be strictly ascending in byte order (term 1)"),
    ([b"ab", b"a"], [0, 1], None, "column 0: terms must be strictly ascending in byte order (term 1)"),
    ([b"\xc3\xa9", b"z"], [0, 1], None, "column 0: terms must be strictly ascending in byte order (term 1)"),
    ([b"a", b"b"], [0, 2], None, "column 0: ordinal out of range (value 1)"),
    ([b"a", b"b"], [-2, 0], None, "column 0: ordinal out of range (value 0)"),
    ([b"a", b"b"], [-1, 0], [0, 1, 2], "column 0: ordinal out of range (value 0)"),
    ([b"a", b"b"], [1, 0], [0, 2, 2], "column 0: the ordinals of a doc must be strictly ascending (doc 0)"),
    ([b"a", b"b"], [0, 0], [0, 2, 2], "column 0: the ordinals of a doc must be strictly ascending (doc 0)"),
    ([b"a", b"b"], [0, 1], [1, 2, 2], "column 0: doc_offsets[0] must be 0"),
    ([b"a", b"b"], [0, 1], [0, 2, 1], "column 0: doc offsets descend"),
])
def test_invalid_columns(lib, terms, ords, offsets, msg):
    assert check(lib, 2, column(terms, ords, offsets)) == (INVALID, "nrtgpu_index_add_keyword_columns: " + msg)


def test_bad_offsets_and_flags(lib):
    c, keep = column([b"a", b"b"], [0, 1])
    bad = np.array([0, 2, 1], np.int64)
    c.term_offsets = bad.ctypes.data
    assert check(lib, 2, (c, keep)) == (INVALID, "nrtgpu_index_add_keyword_columns: column 0: term offsets descend")
    c2, keep2 = column([b"a"], [0, 0])
    start = np.array([1, 1], np.int64)
    c2.term_offsets = start.ctypes.data
    assert check(lib, 2, (c2, keep2)) == (INVALID, "nrtgpu_index_add_keyword_columns: column 0: term_offsets[0] must be 0")
    c3, keep3 = column([b"a"], [0, 0])
    c3.multi_valued = 2
    assert check(lib, 2, (c3, keep3)) == (INVALID, "nrtgpu_index_add_keyword_columns: column 0: multi_valued must be 0 or 1")
    c4, keep4 = column([b"a"], [0, 0])
    c4.ords = None
    assert check(lib, 2, (c4, keep4)) == (INVALID, "nrtgpu_index_add_keyword_columns: column 0: NULL ords")
    assert check(lib, 2, column([b"a"], [0, 0]), column([b"a"], [0, 1])) == \
        (INVALID, "nrtgpu_index_add_keyword_columns: column 1: ordinal out of range (value 1)")
