"""The keyword terms reference (tests/keyword_aggs_reference.py) pinned to the reference's known answers
(OrdinalTermsCollectorManagerTest over the 100 docs of TermsCollectorManagerTestsBase, indexed 10 per segment), plus the
rules the known answers do not show: byte-order ties, a doc in several buckets for the nested collectors, and the union
of leaf dictionaries."""
import numpy as np
import pytest

import keyword_aggs_reference as kr
from nrtsearch_b200.index import HostShard, KeywordColumn, TextField

N = 100


def _order(i):
    v = i // 10 + i % 10
    return v if v < 10 else -1


# the fields of TermsCollectorManagerTestsBase / OrdinalTermsCollectorManagerTest.getIndexRequest, as Lucene stores them
VALUE = KeywordColumn.from_values([str(i % 3) for i in range(N)], False)
VALUE_ORDER = KeywordColumn.from_values([str(_order(i)) for i in range(N)], False)
VALUE_MULTI = KeywordColumn.from_values([[str(i % 2), str(i % 5)] for i in range(N)], True)
VALUE_MULTI_ORDER = KeywordColumn.from_values([[str(_order(i)), str(int(np.fmod(_order(i), 3)))] for i in range(N)], True)   # (Java's %)
SPARSE = KeywordColumn.from_values([str(i // 10) if i % 2 == 0 else None for i in range(N)], False)
ALL = np.ones(N, bool)
RANGE = (np.arange(N) >= 41) & (np.arange(N) <= 50)          # doRangeQuery: int_field in [41, 50]
ORDER_RANGE = (np.arange(N) >= 21) & (np.arange(N) <= 100)   # doOrderRangeQuery: int_field in [21, 100]


def buckets(col, match, size, desc=True):
    r = kr.terms(col, match, size, desc)
    return r["total_buckets"], r["n"], r["other_counts"], list(zip(r["keys"], r["counts"].tolist()))


def unordered(pairs):
    """{count: set of keys}: the reference's assertResponse leaves the order of equal counts open"""
    out = {}
    for k, c in pairs:
        out.setdefault(c, set()).add(k)
    return out


def test_single_valued_known_answers():   # testTermsCollection, Subset, GreaterSize (:163-210)
    for size in (3, 10):
        tb, n, other, got = buckets(VALUE, ALL, size)
        assert (tb, n, other) == (3, 3, 0) and unordered(got) == {34: {"0"}, 33: {"1", "2"}}
    assert buckets(VALUE, ALL, 1) == (3, 1, 66, [("0", 34)])


def test_multi_valued_known_answers():    # testTermsMultiCollection, Subset, GreaterSize (:212-255): the set de-duplicates
    for size in (5, 10):
        tb, n, other, got = buckets(VALUE_MULTI, ALL, size)
        assert (tb, n, other) == (5, 5, 0) and unordered(got) == {60: {"0", "1"}, 20: {"2", "3", "4"}}
    tb, n, other, got = buckets(VALUE_MULTI, ALL, 2)
    assert (tb, n, other) == (5, 2, 60) and unordered(got) == {60: {"0", "1"}}


def test_range_known_answers():           # testTermsRange*, testTermsMultiRange* (:257-330)
    tb, n, other, got = buckets(VALUE, RANGE, 3)
    assert (tb, n, other) == (3, 3, 0) and unordered(got) == {4: {"2"}, 3: {"0", "1"}}
    assert buckets(VALUE, RANGE, 1) == (3, 1, 6, [("2", 4)])
    tb, n, other, got = buckets(VALUE_MULTI, RANGE, 5)
    assert (tb, n, other) == (5, 5, 0) and unordered(got) == {6: {"0", "1"}, 2: {"2", "3", "4"}}
    tb, n, other, got = buckets(VALUE_MULTI, RANGE, 2)
    assert (tb, n, other) == (5, 2, 6) and unordered(got) == {6: {"0", "1"}}


def test_sparse_known_answers():          # testSparseTerms: docs without a value count nowhere
    tb, n, other, got = buckets(SPARSE, RANGE, 3)
    assert (tb, n, other) == (2, 2, 0) and got == [("4", 4), ("5", 1)]


ORDER_DESC = [("-1", 45), ("9", 10), ("8", 9), ("7", 8), ("6", 7), ("5", 6), ("4", 5), ("3", 4), ("2", 3), ("1", 2), ("0", 1)]
MULTI_DESC = [("-1", 45), ("0", 22), ("2", 18), ("1", 15), ("9", 10), ("8", 9), ("7", 8), ("6", 7), ("5", 6), ("4", 5), ("3", 4)]
RANGE_MULTI_DESC = [("-1", 44), ("0", 15), ("2", 11), ("1", 9), ("9", 8), ("8", 7), ("7", 6), ("6", 5), ("5", 4), ("4", 3), ("3", 2)]


def test_ordered_known_answers():         # the _order tests (base :256-420, ORDINAL_EXPECTED_* :38-106): distinct counts
    for size in (11, 20):
        assert buckets(VALUE_ORDER, ALL, size) == (11, 11, 0, ORDER_DESC)
        assert buckets(VALUE_ORDER, ALL, size, False) == (11, 11, 0, ORDER_DESC[::-1])
        assert buckets(VALUE_MULTI_ORDER, ALL, size) == (11, 11, 0, MULTI_DESC)
        assert buckets(VALUE_MULTI_ORDER, ALL, size, False) == (11, 11, 0, MULTI_DESC[::-1])
    assert buckets(VALUE_ORDER, ALL, 2) == (11, 2, 45, ORDER_DESC[:2])
    assert buckets(VALUE_ORDER, ALL, 2, False) == (11, 2, 97, ORDER_DESC[::-1][:2])
    assert buckets(VALUE_MULTI_ORDER, ALL, 2) == (11, 2, 82, MULTI_DESC[:2])
    assert buckets(VALUE_MULTI_ORDER, ALL, 2, False) == (11, 2, 140, MULTI_DESC[::-1][:2])
    assert buckets(VALUE_MULTI_ORDER, ORDER_RANGE, 11) == (11, 11, 0, RANGE_MULTI_DESC)
    assert buckets(VALUE_MULTI_ORDER, ORDER_RANGE, 11, False) == (11, 11, 0, RANGE_MULTI_DESC[::-1])
    assert buckets(VALUE_MULTI_ORDER, ORDER_RANGE, 2) == (11, 2, 55, RANGE_MULTI_DESC[:2])
    assert buckets(VALUE_MULTI_ORDER, ORDER_RANGE, 2, False) == (11, 2, 109, RANGE_MULTI_DESC[::-1][:2])


def test_ties_go_to_the_smaller_term_in_byte_order():
    # "B" < "a" < "é" (0xc3 0xa9) < "\U0001f600" (0xf0 ...) as unsigned bytes; every term counts 1
    col = KeywordColumn.from_values(["\U0001f600", "a", "é", "B"], False)
    assert col.terms == [b"B", b"a", "é".encode(), "\U0001f600".encode()]
    assert buckets(col, np.ones(4, bool), 2) == (4, 2, 2, [("B", 1), ("a", 1)])
    assert buckets(col, np.ones(4, bool), 2, False) == (4, 2, 2, [("B", 1), ("a", 1)])


def test_repeated_terms_of_a_doc_count_once():
    col = KeywordColumn.from_values([["x", "x", "y"], ["y", "y"], []], True)
    assert col.offsets.tolist() == [0, 2, 3, 3] and buckets(col, np.ones(3, bool), 5) == (2, 2, 0, [("y", 2), ("x", 1)])


def test_nested_collectors_see_a_doc_in_each_of_its_buckets():
    n = 6
    sh = HostShard(n_docs=n, doc_base=100, term_off=np.zeros(1, np.int64), post_docs=np.zeros(0, np.int32),
                   post_freqs=np.zeros(0, np.int32), fields=[TextField(None, n, 0)],
                   columns=[np.array([5, 1, 7, 3, 9, 2], np.int64)], column_has=[None])
    col = KeywordColumn.from_values([["a", "b"], ["a"], ["b", "c"], [], ["a", "b", "c"], ["c"]], True)
    scores = np.array([1.0, 3.0, 2.0, 9.0, 0.5, 2.0], np.float32)
    r = kr.terms_nested(sh, col, np.ones(n, bool), 3, True, {"mx": ("max", 0, 0), "s": ("sum", 0, 0), "th": ("top_hits", 2, 0)},
                        scores=scores)
    assert r["keys"] == ["a", "b", "c"] and r["counts"].tolist() == [3, 3, 3] and r["other_counts"] == 0
    assert [v for v, _ in r["nested"]["mx"]] == [9.0, 9.0, 9.0]
    assert [v for v, _ in r["nested"]["s"]] == [15.0, 21.0, 18.0]
    (d, s, t) = r["nested"]["th"][0]
    assert d.tolist() == [101, 100] and t == 3     # bucket "a": docs 0, 1, 4 by score 1.0, 3.0, 0.5
    r = kr.terms_nested(sh, col, np.ones(n, bool), 1, False, {"mx": ("min", 0, 0)}, order_by="mx")
    assert r["keys"] == ["a"] and [v for v, _ in r["nested"]["mx"]] == [1.0]


@pytest.mark.parametrize("multi", [False, True])
def test_union_of_leaf_dictionaries(multi):
    rng = np.random.default_rng(7)
    words = [f"t{i:03d}" for i in range(40)]
    if multi:
        vals = [list(rng.choice(words[: 10 + d // 10], rng.integers(0, 4))) for d in range(300)]
    else:
        vals = [None if d % 7 == 0 else words[rng.integers(0, 10 + d // 10)] for d in range(300)]
    whole = KeywordColumn.from_values(vals, multi)
    leaves = [whole.doc_range(0, 90), whole.doc_range(90, 200), whole.doc_range(200, 300)]
    assert len({len(l.terms) for l in leaves}) == 3            # every leaf numbers its own dictionary
    assert kr.union(leaves) == whole.terms
    g = kr.global_column(leaves)
    assert g.ords.tolist() == whole.ords.tolist()
    if multi:
        assert g.offsets.tolist() == whole.offsets.tolist()
    match = rng.random(300) < 0.6
    assert buckets(g, match, 2048) == buckets(whole, match, 2048)
