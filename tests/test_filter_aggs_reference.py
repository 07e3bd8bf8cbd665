"""The filter-collector reference (tests/filter_aggs_reference.py), the checker of nrtgpu_search_bool_aggs_filtered, pinned on
the CPU: the known answers of FilterCollectorManagerTest.java:86-176 and :572-640 (query_field >= 2 over 14 docs with a
multi-valued value field, filtered by the set {2, 3} or by the same set as a query), value-set equality by bits (-0.0 /
NaN), filters under filters, the empty set and a MUST_NOT-only filter query."""
import math

import numpy as np

import filter_aggs_reference as fr
import oracle
from helpers import shard_from_token_docs
from nrtsearch_b200.search import (BooleanQuery, MatchAllDocsQuery, Occur, RangeQuery, compile_queries, double_to_sortable_long,
                                   float_to_sortable_int)

QUERY_FIELD, VALUE = 0, 1


def known_shard():
    """FilterCollectorManagerTest.addDocuments: query_field 1 with value 0..6; 2 with 1, 2; 3 with {0, 2}, {3, 5}, {4};
    4 with 4, 5 (value is multi-valued)"""
    qf = [1] * 7 + [2] * 2 + [3] * 3 + [4] * 2
    vals = [[v] for v in range(7)] + [[1], [2]] + [[0, 2], [3, 5], [4]] + [[4], [5]]
    sh, _ = shard_from_token_docs([[["x"]] * len(qf)], columns=[np.array(qf, np.int64), np.zeros(len(qf), np.int64)])
    sh.columns[VALUE] = np.array([v for d in vals for v in d], np.int64)
    sh.column_offsets = [None, np.concatenate([[0], np.cumsum([len(d) for d in vals])]).astype(np.int64)]
    return sh


def match_of(sh, query):
    carr, _, qarr, _ = compile_queries([query])
    return oracle.match_bitmap(oracle.OracleIndex(sh), carr, qarr, 0).astype(bool)


QUERY = RangeQuery(QUERY_FIELD, 2, 2**63 - 1)
NESTED = {"nested_terms": ("terms", QUERY_FIELD, 10, True, {}, None)}


def check_known(got):
    assert got["doc_count"] == 3
    t = got["nested_terms"]
    assert (t["n"], t["total_buckets"], t["other_counts"]) == (2, 2, 0)
    assert dict(zip(t["keys"][:2].tolist(), t["counts"][:2].tolist())) == {2: 1, 3: 2}


def test_known_answer_value_set():
    sh = known_shard()
    match = match_of(sh, QUERY)
    assert match.sum() == 7
    check_known(fr.filter_result(sh, match & fr.value_set_mask(sh, VALUE, [2, 3]), NESTED))


def test_known_answer_query_filter():
    sh = known_shard()
    f = BooleanQuery().add(RangeQuery(VALUE, 2, 2), Occur.SHOULD).add(RangeQuery(VALUE, 3, 3), Occur.SHOULD)
    carr, _, qarr, _ = compile_queries([f])
    check_known(fr.filter_result(sh, match_of(sh, QUERY) & fr.query_mask(oracle.OracleIndex(sh), carr, qarr, 0), NESTED))


def test_known_answer_nested_metrics_and_top_hits():
    # :312-370 nests top hits directly under a filter: the filtered docs by score
    sh = known_shard()
    sel = match_of(sh, QUERY) & fr.value_set_mask(sh, VALUE, [3, 2])
    scores = np.linspace(1.0, 2.0, sh.n_docs).astype(np.float32)
    got = fr.filter_result(sh, sel, {"max_qf": ("max", QUERY_FIELD, 0), "sum_qf": ("sum", QUERY_FIELD, 0),
                                     "hits": ("top_hits", 2, 0)}, scores)
    assert got["max_qf"][0] == 3.0 and got["sum_qf"][0] == 8.0
    docs, sc, total = got["hits"]
    assert docs.tolist() == [10, 9] and total == 3 and sc.tolist() == scores[[10, 9]].tolist()


def test_value_set_compares_bits():
    floats = [0.0, -0.0, math.nan, 1.5, -math.inf]
    sh, _ = shard_from_token_docs([[["x"]] * 5], columns=[np.array([float_to_sortable_int(x) for x in floats], np.int64),
                                                          np.array([double_to_sortable_long(x) for x in floats], np.int64)])
    for col, enc in ((0, float_to_sortable_int), (1, double_to_sortable_long)):
        assert fr.value_set_mask(sh, col, [enc(-0.0)]).tolist() == [False, True, False, False, False]
        assert fr.value_set_mask(sh, col, [enc(0.0)]).tolist() == [True, False, False, False, False]
        assert fr.value_set_mask(sh, col, [enc(math.nan), enc(math.nan)]).tolist() == [False, False, True, False, False]
        assert fr.value_set_mask(sh, col, [enc(-math.inf), enc(1.5)]).tolist() == [False, False, False, True, True]


def test_missing_values_and_empty_set():
    sh, _ = shard_from_token_docs([[["x"]] * 4], columns=[np.array([7, 7, 8, 0], np.int64)])
    sh.column_has = [np.array([1, 0, 1, 1], np.uint8)]
    assert fr.value_set_mask(sh, 0, [7, 0]).tolist() == [True, False, False, True]   # a doc without a value never passes
    assert not fr.value_set_mask(sh, 0, []).any()
    got = fr.filter_result(sh, np.ones(4, bool) & fr.value_set_mask(sh, 0, []), {"m": ("min", 0, 0)})
    assert got["doc_count"] == 0 and got["m"][0] == 1.7976931348623157e308   # the unset value


def test_chains():
    sh = known_shard()
    match = match_of(sh, MatchAllDocsQuery())
    outer = fr.value_set_mask(sh, VALUE, [2, 3, 4])
    inner = fr.value_set_mask(sh, QUERY_FIELD, [3, 4])
    got = fr.filter_result(sh, match & outer, {"inner": ("filter", inner, {"t": ("terms", QUERY_FIELD, 5, True, {}, None)})})
    # value in {2, 3, 4}: docs 2, 3, 4, 8, 9 ({0, 2}), 10 ({3, 5}), 11 ({4}), 12 (4)
    assert got["doc_count"] == 8
    assert got["inner"]["doc_count"] == 4
    t = got["inner"]["t"]
    assert dict(zip(t["keys"][:t["n"]].tolist(), t["counts"][:t["n"]].tolist())) == {3: 3, 4: 1}


def test_must_not_only_and_empty_filter_queries_match_nothing():
    sh = known_shard()
    oix = oracle.OracleIndex(sh)
    carr, _, qarr, _ = compile_queries([BooleanQuery().add(RangeQuery(VALUE, 2, 3), Occur.MUST_NOT), BooleanQuery()])
    assert not fr.query_mask(oix, carr, qarr, 0).any()
    assert not fr.query_mask(oix, carr, qarr, 1).any()
