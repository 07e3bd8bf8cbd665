"""Multi-phrase leaves on the host (no GPU): compile_tree's kind-6 clauses and the product's tree compiler (batch_plan.inc
compile_tree) through the multi-phrase planner harness (tests/csrc/multi_phrase_plan_harness.cpp) -- one slot per
position, the weight rule, the one-position rewrite, unions deduplicated over a batch, and every refusal
nrtgpu_search_tree_phrases documents for NRTGPU_MULTI_PHRASE."""
import numpy as np
import pytest

import multi_phrase_plan_harness as mp
import oracle
import phrase_plan_harness as pp
import plan_harness as ph
from nrtsearch_b200 import NrtGpuUnsupported
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, ConstantScoreQuery, MatchPhrasePrefixQuery, MultiPhraseQuery, Occur,
                                   PhraseQuery, TermQuery, compile_tree)

INVALID, UNSUPPORTED = 1, 3
N_TERMS = 200
N_DOCS = 1_000_000
S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
UNION = -2   # DevClause.plane of a union slot (batch_plan.h kUnionList)


@pytest.fixture(scope="module")
def d(built):
    lens = 10 + (np.arange(N_TERMS) * 37) % 500
    off = np.zeros(N_TERMS + 1, np.int64)
    off[1:] = np.cumsum(lens)
    df = lens.astype(np.int64).copy()
    df[189] = 0   # a term without docs in the reader
    return ph.Dictionary(N_DOCS, off, term_field=np.array([0] * 190 + [1] * 10, np.int32), term_df=df,
                         field_doc_count=np.array([N_DOCS, N_DOCS // 2], np.int64))


def term_pos(d):
    """each posting holds 2 positions"""
    return np.concatenate([[0], np.cumsum(2 * np.diff(d.term_off))]).astype(np.int64)


def plan(d, queries, positions=True, cap=0):
    return mp.plan_compiled(d, *compile_tree(queries, phrase_table=True), term_pos=term_pos(d) if positions else None,
                            max_union_postings=cap)


def idf(d, t):
    return float(oracle.bm25_idf(int(d.term_df[t]), int(d.field_doc_count[d.term_field[t]])))


def test_compile_tree_kind_6():
    carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(
        [MultiPhraseQuery([[1, 2], [3]], [0, 2], slop=1), MatchPhrasePrefixQuery([[4]], [5, 6]), MatchPhrasePrefixQuery([[4]], [])],
        phrase_table=True)
    assert [carr[i].kind for i in range(ncl)] == [6, 6, 6]
    assert [(tarr[i].term, tarr[i].position) for i in range(n_pt)] == [(1, 0), (2, 0), (3, 2), (4, 0), (5, 1), (6, 1)]
    assert (parr[0].slop, parr[2].term_begin, parr[2].term_end) == (1, 6, 6)   # no expansion: no terms
    with pytest.raises(NrtGpuUnsupported):
        compile_tree([MultiPhraseQuery([[1, 2]])])
    with pytest.raises(ValueError):
        MultiPhraseQuery([[1], [2]], [0, 0]).term_positions()
    assert MultiPhraseQuery([[1], []]).term_positions() == []


def test_one_slot_per_position_and_the_weight(d):
    q = BoostQuery(MultiPhraseQuery([[1], [2, 3, 189], [4]], slop=0), 2.0)
    p = plan(d, [q])
    cl = p.query_clauses(0)
    rec = p.phrases[0]
    assert rec["n_terms"] == 3 and list(rec["offset"][:3]) == [0, 1, 2]
    terms = cl[rec["clause0"]:rec["clause0"] + 3]
    assert list(terms["slot"]) == [0, 1, 2]
    assert list(terms["plane"] == UNION) == [False, True, False]
    assert list(terms["col"][[0, 2]]) == [1, 4]
    assert p.unions() == [[2, 3, 189]] and list(p.union_mode) == [2]
    s = sum(idf(d, t) for t in (1, 2, 3, 4))   # 189 has df 0: no idf
    assert rec["weight"] == np.float32(np.float32(2.0) * np.float32(s))
    assert cl[0]["kind"] == 4 and cl[0]["weight"] == rec["weight"]
    assert p.union_postings == sum(int(d.term_off[t + 1] - d.term_off[t]) for t in (2, 3, 189))
    assert p.union_positions == 2 * p.union_postings


def test_one_position_is_a_scored_union_slot(d):
    p = plan(d, [BoostQuery(MatchPhrasePrefixQuery([], [7, 5, 6]), 1.5)], positions=False)
    (c,) = p.query_clauses(0)
    assert (c["kind"], c["plane"], c["slot"], c["scoring"]) == (0, UNION, 0, 1)
    assert p.unions() == [[5, 6, 7]] and list(p.union_mode) == [1]   # ascending term id
    want = [np.float32(1.5) * np.float32(oracle.bm25_idf(int(d.term_df[t]), N_DOCS)) for t in (5, 6, 7)]
    assert p.union_weight.tolist() == [float(w) for w in want]
    assert p.queries[0]["req_term_mask"] == 1 and p.queries[0]["driver_mask"] == 1
    # under FILTER or a ConstantScoreQuery it only has to match: a presence union
    p = plan(d, [BooleanQuery().add(TermQuery(1), M).add(MatchPhrasePrefixQuery([], [5, 6]), F),
                 ConstantScoreQuery(MatchPhrasePrefixQuery([], [5, 6]))], positions=False)
    assert p.unions() == [[5, 6]] and list(p.union_mode) == [0]
    assert len(p.union_clause) == 2


def test_degenerate_multi_phrases(d):
    p = plan(d, [MatchPhrasePrefixQuery([], [9]), MatchPhrasePrefixQuery([[1]], []), MultiPhraseQuery([[1], [189]])])
    (c0,), (c1,) = p.query_clauses(0), p.query_clauses(1)
    assert (c0["kind"], c0["plane"]) != (0, UNION) and c0["kind"] == 0   # one alternative: that TermQuery
    assert c0["post_base"] == d.term_off[9] and c0["weight"] == np.float32(oracle.bm25_idf(int(d.term_df[9]), N_DOCS))
    assert (c1["kind"], c1["col"]) == (4, -1)   # no expansion: a phrase of no terms, matches nothing
    assert p.queries[1]["empty"] == 1
    assert len(p.phrases) == 1 and p.union_postings == 0   # [1] [189]: both single terms, no union


def test_unions_are_deduplicated_over_the_batch(d):
    qs = [MatchPhrasePrefixQuery([[i % 5]], [10, 11, 12] if i % 2 else [12, 11, 10]) for i in range(64)] + \
         [MatchPhrasePrefixQuery([], [10, 11, 12]), BoostQuery(MatchPhrasePrefixQuery([], [10, 11, 12]), 2.0)]
    p = plan(d, qs)
    assert p.unions() == [[10, 11, 12]] * 3   # a phrase position, and one scored union per boost
    assert sorted(p.union_mode.tolist()) == [1, 1, 2]
    assert len(p.union_clause) == 66
    assert p.union_postings == 3 * sum(int(d.term_off[t + 1] - d.term_off[t]) for t in (10, 11, 12))


def test_slot_counting(d):
    six = BooleanQuery()
    for t in range(6):
        six.add(TermQuery(t), S)
    ok = BooleanQuery(list(six.clauses)).add(MultiPhraseQuery([[10, 11, 12, 13], list(range(20, 60))]), S)
    p = plan(d, [ok])
    assert p.queries[0]["n_term"] == 8
    with pytest.raises(ph.PlanError) as e:
        plan(d, [BooleanQuery(list(ok.clauses)).add(TermQuery(7), S)])
    assert e.value.rc == UNSUPPORTED and "more than 8" in str(e.value)
    with pytest.raises(ph.PlanError) as e:
        plan(d, [BooleanQuery(list(six.clauses)).add(PhraseQuery([1, 2]), S).add(MatchPhrasePrefixQuery([], [3, 4]), S)])
    assert e.value.rc == UNSUPPORTED and "more than 8 term slots" in str(e.value)


@pytest.mark.parametrize("q,positions,code,msg", [
    (MultiPhraseQuery([[1], list(range(0, 129))]), True, UNSUPPORTED, "more than 128 terms at one position"),
    (MultiPhraseQuery([[1, 2], [3, 1]], slop=1), True, UNSUPPORTED, "sloppy phrase with a repeated term"),
    (MultiPhraseQuery([[1], [195]]), True, INVALID, "same field"),
    (MultiPhraseQuery([[1], [2]], [3, 1]), True, INVALID, "positions must be added in order"),
    (MultiPhraseQuery([[1], [2]], [-1, 0]), True, INVALID, "positions must be >= 0"),
    (MultiPhraseQuery([[1], [2]], slop=-1), True, INVALID, "slop must be >= 0"),
    (MultiPhraseQuery([[1], [N_TERMS]]), True, INVALID, "phrase term id out of range"),
    (MultiPhraseQuery([[1], [2, 3]]), False, INVALID, "without position data"),
])
def test_refusals(d, q, positions, code, msg):
    with pytest.raises(ph.PlanError) as e:
        plan(d, [q], positions=positions)
    assert e.value.rc == code and msg in str(e.value)


def test_a_repeat_at_one_position_is_no_sloppy_repeat(d):
    plan(d, [MultiPhraseQuery([[1, 1], [2]], slop=2)])
    plan(d, [MatchPhrasePrefixQuery([], list(range(128)))], positions=False)   # 128 alternatives and no positions: fine


def test_union_postings_cap(d):
    q = MatchPhrasePrefixQuery([], [10, 11])
    n = sum(int(d.term_off[t + 1] - d.term_off[t]) for t in (10, 11))
    plan(d, [q], cap=n)
    with pytest.raises(ph.PlanError) as e:
        plan(d, [q], cap=n - 1)
    assert e.value.rc == UNSUPPORTED and f"gather {n} postings, more than {n - 1}" in str(e.value)


def test_other_entry_points_refuse_kind_6(d):
    """without the union entry points' flag (flat batches, tree rescoring) kind 6 is a bad clause kind"""
    arrays = compile_tree([MatchPhrasePrefixQuery([[1]], [2, 3])], phrase_table=True)
    with pytest.raises(ph.PlanError) as e:
        pp.plan_compiled(d, *arrays)
    assert e.value.rc == INVALID and "bad clause kind" in str(e.value)


def test_union_positions_cap(d):
    """an image whose terms hold 2^26 positions each: two alternatives of a phrase position pass the 2^27 positions cap,
    three do not (a one-position leaf merges no positions)"""
    big = np.arange(N_TERMS + 1, dtype=np.int64) << 26
    arrays = lambda alts: compile_tree([MultiPhraseQuery([[1], alts])], phrase_table=True)   # noqa: E731
    assert mp.plan_compiled(d, *arrays([2, 3]), term_pos=big).union_positions == 1 << 27
    with pytest.raises(ph.PlanError) as e:
        mp.plan_compiled(d, *arrays([2, 3, 4]), term_pos=big)
    assert e.value.rc == UNSUPPORTED and f"merge {3 << 26} positions, more than {1 << 27}" in str(e.value)
    p = mp.plan_compiled(d, *compile_tree([MatchPhrasePrefixQuery([], [2, 3, 4])], phrase_table=True), term_pos=big)
    assert p.union_positions == 0


def test_repeated_terms_count_in_the_weight(d):
    p = plan(d, [MatchPhrasePrefixQuery([[5]], [4, 5, 6])])
    s = idf(d, 5) + idf(d, 4) + idf(d, 5) + idf(d, 6)   # position 0, then position 1 in ascending term id
    assert p.phrases[0]["weight"] == np.float32(s)
