"""The nested-collector reference (tests/nested_aggs_reference.py), the checker of nrtgpu_search_bool_aggs_nested, pinned on
the CPU against the reference's known answers: NestedCollectorOrderTest.java:60-235 (buckets of int_field ordered by a
nested max of value_field_2, with and without a second nested max, over every doc and over int_field in [2, 4]) and the
structure of NestedCollectionTest.java:124-192 (two buckets of 50 docs, top 5 hits each, totalHits 50), with a BM25 query in
place of the script score."""
import math

import numpy as np
import pytest

import nested_aggs_reference as nr
import oracle
from helpers import shard_from_token_docs
from nrtsearch_b200.search import MatchAllDocsQuery, RangeQuery, TermQuery, compile_queries

INT_FIELD, VALUE, VALUE_2 = 0, 1, 2


def order_shard():
    """NestedCollectorOrderTest.initIndex: doc (i, j), i in 1..5, j in 1..20: int_field i, value_field i*j, value_field_2 -i*j"""
    i, j = np.repeat(np.arange(1, 6), 20), np.tile(np.arange(1, 21), 5)
    sh, _ = shard_from_token_docs([[["x"]] * 100], columns=[i.astype(np.int64), (i * j).astype(np.int64), (-i * j).astype(np.int64)])
    return sh


def run(sh, query, size, desc, extra=False):
    carr, _, qarr, _ = compile_queries([query])
    match = oracle.match_bitmap(oracle.OracleIndex(sh), carr, qarr, 0).astype(bool)
    nested = {"max_order": ("max", VALUE_2, 0)}
    if extra:
        nested["additional"] = ("max", VALUE, 0)
    return nr.terms_nested(sh, match, INT_FIELD, size, desc, nested, order_by="max_order")


ALL = MatchAllDocsQuery()     # the exists query matches every doc
RANGE = RangeQuery(INT_FIELD, 2, 4)


@pytest.mark.parametrize("query, size, desc, total, n, other, keys", [
    (ALL, 5, True, 5, 5, 0, [1, 2, 3, 4, 5]),          # testNestedOrder
    (ALL, 5, False, 5, 5, 0, [5, 4, 3, 2, 1]),
    (ALL, 2, True, 5, 2, 60, [1, 2]),                  # testNestedOrderSubset
    (ALL, 2, False, 5, 2, 60, [5, 4]),
    (ALL, 10, True, 5, 5, 0, [1, 2, 3, 4, 5]),         # testNestedOrderGreaterSize
    (ALL, 10, False, 5, 5, 0, [5, 4, 3, 2, 1]),
    (RANGE, 3, True, 3, 3, 0, [2, 3, 4]),              # testRangeNestedOrder
    (RANGE, 3, False, 3, 3, 0, [4, 3, 2]),
    (RANGE, 2, True, 3, 2, 20, [2, 3]),                # testRangeNestedOrderSubset
    (RANGE, 2, False, 3, 2, 20, [4, 3]),
    (RANGE, 10, True, 3, 3, 0, [2, 3, 4]),             # testRangeNestedOrderGreaterSize
    (RANGE, 10, False, 3, 3, 0, [4, 3, 2]),
])
def test_nested_order_known_answers(query, size, desc, total, n, other, keys):
    got = run(order_shard(), query, size, desc)
    assert (got["total_buckets"], got["n"], got["other_counts"]) == (total, n, other)
    assert got["keys"][:n].tolist() == keys and got["counts"][:n].tolist() == [20] * n
    assert [v for v, _ in got["nested"]["max_order"]] == [-float(k) for k in keys]


@pytest.mark.parametrize("query, size, keys, additional", [
    (ALL, 5, [1, 2, 3, 4, 5], [20.0, 40.0, 60.0, 80.0, 100.0]),   # testNestedOrderWithAdditionalCollector
    (RANGE, 3, [2, 3, 4], [40.0, 60.0, 80.0]),                    # testRangeNestedOrderWithAdditionalCollector
])
def test_nested_order_with_additional_collector(query, size, keys, additional):
    sh = order_shard()
    desc = run(sh, query, size, True, extra=True)
    asc = run(sh, query, size, False, extra=True)
    assert desc["keys"][:size].tolist() == keys and asc["keys"][:size].tolist() == keys[::-1]
    assert [v for v, _ in desc["nested"]["additional"]] == additional
    assert [v for v, _ in asc["nested"]["additional"]] == additional[::-1]


def collection_shard():
    """NestedCollectionTest's 100 docs (int_field_2 = id % 2) with a text field where doc id holds 'a' 1 + id // 10 times in
    ten tokens, so a TermQuery('a') scores by id // 10 and every group of ten ids ties"""
    docs = [["a"] * (1 + d // 10) + ["b"] * (9 - d // 10) for d in range(100)]
    ids = np.arange(100, dtype=np.int64)
    sh, vocab = shard_from_token_docs([docs], columns=[ids % 2, ids])
    return sh, vocab


def test_nested_top_hits_structure():
    sh, vocab = collection_shard()
    oix = oracle.OracleIndex(sh)
    carr, ncl, qarr, nq = compile_queries([TermQuery(vocab[(0, "a")])])
    match = oracle.match_bitmap(oix, carr, qarr, 0).astype(bool)
    scores = nr.query_scores(sh, oix, carr, qarr, 0, match)
    got = nr.terms_nested(sh, match, 0, 2, True, {"nested": ("top_hits", 5, 0), "paged": ("top_hits", 5, 2)}, scores=scores)
    assert got["n"] == 2 and got["total_buckets"] == 2 and got["other_counts"] == 0
    assert sorted(got["keys"].tolist()) == [0, 1] and got["counts"].tolist() == [50, 50]
    top_docs, top_scores, _, _, _ = oracle.search_compiled(oix, carr, ncl, qarr, nq, 100)
    for b, key in enumerate(got["keys"].tolist()):
        docs, sc, total = got["nested"]["nested"][b]
        assert total == 50 and len(docs) == 5
        assert docs.tolist() == [90 + key, 92 + key, 94 + key, 96 + key, 98 + key]   # tied scores: doc ascending
        assert len(set(sc.tolist())) == 1 and sc[0] == top_scores[0][0]              # the scores of the top-level hits
        assert sc.view(np.uint32).tolist() == [top_scores[0][top_docs[0].tolist().index(d)].view(np.uint32) for d in docs]
        p_docs, _, p_total = got["nested"]["paged"][b]
        assert p_docs.tolist() == docs[2:].tolist() and p_total == 50


def test_top_hits_larger_than_the_bucket_and_score_order():
    sh, vocab = collection_shard()
    oix = oracle.OracleIndex(sh)
    carr, _, qarr, _ = compile_queries([RangeQuery(1, 0, 14)])   # ids 0..14: constant score
    match = oracle.match_bitmap(oix, carr, qarr, 0).astype(bool)
    scores = np.where(match, np.float32(1.0), np.float32(0.0)).astype(np.float32)
    scores[3] = np.float32(2.0)
    got = nr.terms_nested(sh, match, 0, 2, True, {"h": ("top_hits", 100, 1)}, scores=scores)
    assert got["counts"].tolist() == [8, 7] and got["keys"].tolist() == [0, 1]
    d0, _, t0 = got["nested"]["h"][0]
    d1, s1, t1 = got["nested"]["h"][1]
    assert t0 == 8 and d0.tolist() == [2, 4, 6, 8, 10, 12, 14]        # position 0 (doc 0) skipped by start_hit 1
    assert t1 == 7 and d1.tolist() == [1, 5, 7, 9, 11, 13] and s1.tolist() == [1.0] * 6   # doc 3 scores highest


def test_order_by_value_ties_nan_and_signed_zero():
    """Double.compare order: NaN above +inf, -0.0 below 0.0; equal values go to the smaller key in both directions"""
    keys = [10, 20, 30, 40, 50, 60]
    values = [1.0, math.nan, -0.0, 0.0, 1.0, math.inf]
    counts = [1] * 6
    assert [keys[b] for b in nr.order_buckets(keys, counts, 6, True, values)] == [20, 60, 10, 50, 40, 30]
    assert [keys[b] for b in nr.order_buckets(keys, counts, 6, False, values)] == [30, 40, 10, 50, 60, 20]
    assert [keys[b] for b in nr.order_buckets(keys, [3, 1, 3, 2, 1, 1], 3, True)] == [10, 30, 40]
