"""The keyword query reference (tests/keyword_query_reference.py) pinned on the CPU, and the bounds -> code range rule of the
host compiler (keyword_range_codes in batch_plan.inc, through tests/csrc/keyword_query_harness.cpp) checked against it:
  - AtomFieldTest.rangeQuery (AtomFieldTest.java:455-515): docs a..f, eight bound combinations, on a SORTED and a
    SORTED_SET column;
  - PrefixQueryTest.testAtomPrefixQuery (:98-108): prefix1 -> docs 0-2, prefix2 -> 3-6, prefix -> 0-6, other -> none;
  - FilterCollectorManagerTest.testTextFilterSet (:258-265): the {"2", "3"} set over the text values of the 14-doc index
    whose numeric set's answers tests/test_filter_aggs_reference.py pins;
  - over random dictionaries, the code range of every bound combination selects exactly the reference's terms."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import filter_aggs_reference as fr
import keyword_query_reference as kr
from nrtsearch_b200.index import KeywordColumn

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libkeyword_query_harness.so")
NO_LOWER, NO_UPPER, LOWER_EXCLUSIVE, UPPER_EXCLUSIVE, PREFIX = 1, 2, 4, 8, 16


@pytest.fixture(scope="module")
def lib():
    h = C.CDLL(_PATH)
    h.kqh_last_error.restype = C.c_char_p
    h.kqh_seek.restype = C.c_int64
    h.kqh_seek.argtypes = [C.c_char_p, C.c_void_p, C.c_int32, C.c_char_p, C.c_int32]
    h.kqh_range.argtypes = [C.c_char_p, C.c_void_p, C.c_int32, C.c_char_p, C.c_int32, C.c_char_p, C.c_int32, C.c_int32,
                            C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
    return h


def code_range(lib, terms, lower=None, upper=None, include_lower=True, include_upper=True, prefix=None):
    """[lo, hi] of the compiler's rule on the dictionary `terms` (sorted bytes)"""
    blob = b"".join(terms)
    off = np.concatenate([[0], np.cumsum([len(t) for t in terms])]).astype(np.int64)
    lo, hi = C.c_int64(), C.c_int64()
    if prefix is not None:
        a, b, flags = prefix, b"", PREFIX
    else:
        a, b = lower or b"", upper or b""
        flags = (NO_LOWER if lower is None else 0 if include_lower else LOWER_EXCLUSIVE) | \
                (NO_UPPER if upper is None else 0 if include_upper else UPPER_EXCLUSIVE)
    assert lib.kqh_range(blob, off.ctypes.data, len(terms), a, len(a), b, len(b), flags, C.byref(lo), C.byref(hi)) == 0
    return lo.value, hi.value


def terms_in(terms, lo, hi):
    """the terms whose code 2i + 2 lies in [lo, hi]"""
    return [t for i, t in enumerate(terms) if lo <= 2 * i + 2 <= hi]


# AtomFieldTest.rangeQuery: (lower, upper, lower exclusive, upper exclusive) -> the docs' values that match
ATOM_CASES = [
    ("b", "e", False, False, "bcde"), ("b", "e", True, False, "cde"), ("b", "e", False, True, "bcd"), ("b", "e", True, True, "cd"),
    (None, "d", False, False, "abcd"), (None, "d", False, True, "abc"), ("b", None, False, False, "bcdef"),
    ("b", None, True, False, "cdef"),
]


@pytest.mark.parametrize("multi", [False, True])
@pytest.mark.parametrize("lower,upper,lex,uex,want", ATOM_CASES)
def test_atom_field_range_query(lib, multi, lower, upper, lex, uex, want):
    vals = list("abcdef")
    col = KeywordColumn.from_values([[v] for v in vals] if multi else vals, multi)
    enc = lambda x: None if x is None else x.encode()
    m = kr.match_mask(col, kr.range_pred(enc(lower), enc(upper), not lex, not uex))
    assert "".join(v for v, hit in zip(vals, m) if hit) == want
    lo, hi = code_range(lib, col.terms, enc(lower), enc(upper), not lex, not uex)
    assert "".join(t.decode() for t in terms_in(col.terms, lo, hi)) == want


PREFIX_DOCS = ["prefix1a", "prefix1b", "prefix1c", "prefix2a", "prefix2b", "prefix2c", "prefix2d", "not_prefix1", "not_prefix2"]


@pytest.mark.parametrize("prefix,want", [("prefix1", [0, 1, 2]), ("prefix2", [3, 4, 5, 6]), ("prefix", list(range(7))),
                                         ("other", [])])
def test_atom_prefix_query(lib, prefix, want):
    col = KeywordColumn.from_values(PREFIX_DOCS, False)
    assert np.flatnonzero(kr.match_mask(col, kr.prefix_pred(prefix.encode()))).tolist() == want
    lo, hi = code_range(lib, col.terms, prefix=prefix.encode())
    held = set(terms_in(col.terms, lo, hi))
    assert [d for d, v in enumerate(PREFIX_DOCS) if v.encode() in held] == want


def test_text_filter_set():
    """testTextFilterSet: the text values of FilterCollectorManagerTest's 14 docs filtered by {"2", "3"} give the answers of
    the numeric set {2, 3}"""
    sh = fr_known_shard()
    vals = [[v] for v in range(7)] + [[1], [2]] + [[0, 2], [3, 5], [4]] + [[4], [5]]
    col = KeywordColumn.from_values([[str(v) for v in d] for d in vals], True)
    text = kr.match_mask(col, kr.set_pred([b"2", b"3"]))
    assert np.array_equal(text, fr.value_set_mask(sh, 1, [2, 3]))
    assert np.flatnonzero(text).tolist() == [2, 3, 8, 9, 10]


def fr_known_shard():
    import test_filter_aggs_reference as t
    return t.known_shard()


def _random_terms(rng):
    alphabet = [0x00, 0x01, 0x61, 0x62, 0x7F, 0x80, 0xFE, 0xFF]
    n = rng.choice([0, 1, 2, 5, 20, 60])
    s = {b""} if rng.random() < 0.3 else set()
    while len(s) < n:
        s.add(bytes(rng.choice(alphabet) for _ in range(rng.randint(0, 4))))
    return sorted(s)


def _random_bound(rng, terms):
    r = rng.random()
    if terms and r < 0.4:
        return rng.choice(terms)
    if terms and r < 0.55:   # between / beside held terms
        t = rng.choice(terms)
        return t + bytes([rng.choice([0x00, 0x80, 0xFF])])
    if r < 0.65:
        return b""
    if r < 0.75:
        return b"\xff" * rng.randint(1, 5)   # after every term
    alphabet = [0x00, 0x01, 0x61, 0x62, 0x7F, 0x80, 0xFE, 0xFF]
    return bytes(rng.choice(alphabet) for _ in range(rng.randint(0, 4)))


def test_bounds_rule_random_dictionaries(lib):
    rng = random.Random(20261018)
    for _ in range(400):
        terms = _random_terms(rng)
        for _ in range(10):
            lower, upper = _random_bound(rng, terms), _random_bound(rng, terms)
            if rng.random() < 0.2:
                upper = lower   # equal bounds, both ways exclusive included
            lower = None if rng.random() < 0.15 else lower
            upper = None if rng.random() < 0.15 else upper
            il, iu = rng.random() < 0.5, rng.random() < 0.5
            lo, hi = code_range(lib, terms, lower, upper, il, iu)
            assert 1 <= lo <= 2 * len(terms) + 1 and 1 <= hi <= 2 * len(terms) + 1
            assert terms_in(terms, lo, hi) == kr.matching_terms(terms, kr.range_pred(lower, upper, il, iu)), (terms, lower, upper, il, iu)
            p = _random_bound(rng, terms)[: rng.randint(0, 3)]
            if rng.random() < 0.1:
                p = b"\xff" * rng.randint(1, 3)
            lo, hi = code_range(lib, terms, prefix=p)
            assert terms_in(terms, lo, hi) == kr.matching_terms(terms, kr.prefix_pred(p)), (terms, p)


@pytest.mark.parametrize("prefix", [b"", b"\xff", b"\xff\xff"])
def test_prefix_without_upper_bound(lib, prefix):
    terms = sorted({b"", b"a", b"\xfe", b"\xff", b"\xff\x00", b"\xff\xff", b"\xff\xff\xff"})
    lo, hi = code_range(lib, terms, prefix=prefix)
    assert hi == 2 * len(terms) + 1
    assert terms_in(terms, lo, hi) == [t for t in terms if t.startswith(prefix)]


def test_seek_codes(lib):
    terms = [b"b", b"d"]
    blob, off = b"bd", np.array([0, 1, 2], np.int64)
    seek = lambda t: lib.kqh_seek(blob, off.ctypes.data, 2, t, len(t))
    assert [seek(t) for t in (b"a", b"b", b"c", b"d", b"e")] == [1, 2, 3, 4, 5]
    assert code_range(lib, terms, b"c", b"c") == (3, 3)          # lower > upper after the gap: empty
    assert code_range(lib, terms, b"d", b"b") == (4, 2)          # lower > upper: accepted, matches nothing
    assert code_range(lib, terms, b"b", b"b", False, False) == (3, 1)
