"""Phrase leaves on the host (no GPU): compile_tree's phrase table and the product's tree compiler (batch_plan.inc
compile_tree) through the phrase planner harness (tests/csrc/phrase_plan_harness.cpp) -- slot layout, phrase records,
covers and root masks, degenerate phrases, and every refusal nrtgpu_search_tree_phrases documents."""
import numpy as np
import pytest

import oracle
import phrase_plan_harness as pp
import plan_harness as ph
import tree_plan_harness as th
from nrtsearch_b200 import NrtGpuUnsupported, _native
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, Occur, PhraseQuery, TermQuery, compile_tree)

INVALID, UNSUPPORTED = 1, 3
LENS = [100, 200, 300, 50, 1000, 5, 70, 80, 90, 110]   # postings of terms 0..9; terms 8, 9 are on field 1
N_DOCS = 3_000_000
S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT


@pytest.fixture(scope="module")
def d(built):
    off = np.zeros(len(LENS) + 1, np.int64)
    off[1:] = np.cumsum(LENS)
    return ph.Dictionary(N_DOCS, off, term_field=np.array([0] * 8 + [1] * 2, np.int32),
                         field_doc_count=np.array([N_DOCS, N_DOCS // 2], np.int64))


def plan_arrays(d, *arrays, top_k=10, positions=True):
    """(PhrasePlan, phrase records, [nq + 1] record ranges) of compile_tree(..., phrase_table=True)'s arrays; raises PlanError"""
    p = pp.plan_compiled(d, *arrays, top_k=top_k, positions=positions)
    return p, p.phrases, p.phrase_begin


def plan(d, queries, top_k=10, positions=True):
    return plan_arrays(d, *compile_tree(queries, phrase_table=True), top_k=top_k, positions=positions)


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(TermQuery(c) if isinstance(c, int) else c, o)
    return q


def idf_weight(d, terms, boost=1.0):
    f = int(d.term_field[terms[0]])
    s = 0.0
    for t in terms:
        s += float(oracle.bm25_idf(int(d.term_df[t]), int(d.field_doc_count[f])))
    return np.float32(np.float32(boost) * np.float32(s))


# ---------------------------------------------------------------- compile_tree (Python mirror)

def test_compile_tree_phrase_table():
    q = bq((PhraseQuery([1, 2]), M), (BoostQuery(PhraseQuery([3, 4, 3], positions=[0, 2, 2], slop=1), 2.0), S))
    carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree([q, PhraseQuery([5])], phrase_table=True)
    assert (n_ph, n_pt, nn, nq) == (3, 6, 0, 2)
    assert [(carr[i].kind, carr[i].id, carr[i].boost) for i in range(ncl)] == [(4, 0, 1.0), (4, 1, 2.0), (4, 2, 1.0)]
    assert [(parr[i].term_begin, parr[i].term_end, parr[i].slop) for i in range(3)] == [(0, 2, 0), (2, 5, 1), (5, 6, 0)]
    assert [(tarr[i].term, tarr[i].position) for i in range(6)] == [(1, 0), (2, 1), (3, 0), (4, 2), (3, 2), (5, 0)]
    assert carr[qarr[1].clause_begin].occur == M   # a bare PhraseQuery is the root's one MUST clause
    with pytest.raises(NrtGpuUnsupported):
        compile_tree([q])   # without the phrase table
    with pytest.raises(ValueError):
        PhraseQuery([1, 2], positions=[0]).term_positions()


# ---------------------------------------------------------------- the product's compiler

def test_slot_layout_records_and_root_masks(d):
    q = bq((PhraseQuery([1, 3, 2]), M), (6, S), (BoostQuery(PhraseQuery([4, 5], positions=[0, 2], slop=3), 1.5), S))
    p, recs, begin = plan(d, [q])
    cl = p.query_clauses(0)
    assert list(cl["kind"]) == [4, 0, 4, 0, 0, 0, 0, 0]
    # the root's clauses first, then the phrase terms in position order, one presence-only slot each
    assert list(cl["slot"]) == [-1, 0, -1, 1, 2, 3, 4, 5]
    assert list(cl["col"][[0, 2]]) == [0, 1] and list(cl["col"][3:]) == [1, 3, 2, 4, 5]
    assert not cl["scoring"][3:].any() and (cl["occur"][3:] == F).all()
    assert list(begin) == [0, 2] and len(recs) == 2
    r0, r1 = recs
    assert (r0["clause0"], r0["n_terms"], r0["slop"], r0["field"], list(r0["offset"][:3])) == (3, 3, 0, 0, [0, 1, 2])
    assert r0["cover_slot"] == 2   # term 3: 50 postings
    assert (r1["clause0"], r1["n_terms"], r1["slop"], list(r1["offset"][:2]), r1["cover_slot"]) == (6, 2, 3, [0, 2], 5)
    assert r0["weight"] == idf_weight(d, [1, 3, 2]) and cl["weight"][0] == r0["weight"]
    assert r1["weight"] == idf_weight(d, [4, 5], 1.5)
    qq = p.queries[0]
    assert qq["req_term_mask"] == 0b1110 and qq["not_term_mask"] == 0   # a MUST phrase at the root needs all its terms
    assert qq["driver_mask"] == 1 << 2 and qq["n_term"] == 6 and not qq["empty"]
    assert p.alg_postings == sum(LENS[t] for t in (6, 1, 3, 2, 4, 5))


def test_covers_with_phrases(d):
    dm = DisjunctionMaxQuery([PhraseQuery([4, 2]), PhraseQuery([8, 9])], 0.1)
    p, recs, _ = plan(d, [bq((0, S), (PhraseQuery([1, 5]), S)), bq((dm, M)), bq((PhraseQuery([0, 1]), N), (3, M)),
                          bq((PhraseQuery([1, 2]), F), (bq((0, S), (4, S)), M))])
    slot = lambda q, t: int(p.query_clauses(q)[(p.query_clauses(q)["kind"] == 0) & (p.query_clauses(q)["col"] == t)]["slot"][0])  # noqa
    assert p.queries[0]["driver_mask"] == 1 << 0 | 1 << slot(0, 5)          # SHOULD union: the term and the phrase's rarest
    assert p.queries[1]["driver_mask"] == 1 << slot(1, 2) | 1 << slot(1, 8)  # dismax: each phrase's rarest term
    assert p.queries[2]["driver_mask"] == 1 << 0 and p.queries[2]["not_term_mask"] == 0   # MUST_NOT phrase: no mask
    assert p.queries[3]["driver_mask"] == 1 << slot(3, 1)                    # FILTER phrase (300 + 200) vs 100 + 1000
    assert p.queries[3]["req_term_mask"] == 1 << slot(3, 1) | 1 << slot(3, 2)
    assert [r["n_terms"] for r in recs] == [2, 2, 2, 2, 2]


def test_one_term_and_empty_phrases(d):
    p, recs, _ = plan(d, [bq((BoostQuery(PhraseQuery([4]), 2.0), M), (PhraseQuery([]), S)), bq((PhraseQuery([]), M), (1, S)),
                          bq((PhraseQuery([], slop=2), S), (2, S))])
    assert len(recs) == 0
    c0 = p.query_clauses(0)
    assert (c0[0]["kind"], c0[0]["slot"], c0[0]["scoring"], c0[0]["col"]) == (0, 0, 1, 0)   # the term leaf itself
    assert c0[0]["weight"] == idf_weight(d, [4], 2.0)
    assert (c0[1]["kind"], c0[1]["col"]) == (4, -1) and not p.queries[0]["empty"]
    assert p.queries[0]["driver_mask"] == 1
    assert p.queries[1]["empty"]                                  # a required phrase of no terms matches nothing
    assert not p.queries[2]["empty"] and p.queries[2]["driver_mask"] == 1


def test_without_phrases_it_is_the_tree_compile(d):
    q = [bq((bq((0, S), (1, S)), M), (2, S))]
    p, recs, _ = plan(d, q)
    t = th.plan(d, q, 10)
    assert np.array_equal(p.clauses, t.clauses) and np.array_equal(p.queries, t.queries) and np.array_equal(p.nodes, t.nodes)
    assert len(recs) == 0


def _arrays(clauses, phrases, terms, queries=((0, 1, 0, 0, 0, 0.0),)):
    carr = (_native.Clause * max(len(clauses), 1))(*[_native.Clause(*c) for c in clauses])
    narr = (_native.Node * 1)()
    parr = (_native.Phrase * max(len(phrases), 1))(*[_native.Phrase(*p) for p in phrases])
    tarr = (_native.PhraseTerm * max(len(terms), 1))(*[_native.PhraseTerm(*t) for t in terms])
    qarr = (_native.Query * len(queries))(*[_native.Query(*q) for q in queries])
    return carr, len(clauses), narr, 0, parr, len(phrases), tarr, len(terms), qarr, len(queries)


PH = (1, 4, 0, 1.0, 0, 0)   # a MUST clause of phrase 0
INVALID_PHRASES = [
    ([(1, 4, 1, 1.0, 0, 0)], [(0, 2, 0, 0)], [(1, 0), (2, 1)], "phrase id out of range"),
    ([(1, 4, -1, 1.0, 0, 0)], [(0, 2, 0, 0)], [(1, 0), (2, 1)], "phrase id out of range"),
    ([PH], [(0, 2, 0, 0)], [(1, 0), (99, 1)], "phrase term id out of range"),
    ([PH], [(0, 3, 0, 0)], [(1, 0), (2, 1)], "phrase term range out of bounds"),
    ([PH], [(2, 1, 0, 0)], [(1, 0), (2, 1)], "phrase term range out of bounds"),
    ([PH], [(-1, 1, 0, 0)], [(1, 0), (2, 1)], "phrase term range out of bounds"),
    ([PH], [(0, 2, 0, 0)], [(1, 0), (8, 1)], "same field"),
    ([PH], [(0, 2, 0, 0)], [(1, -1), (2, 0)], "positions must be >= 0"),
    ([PH], [(0, 2, 0, 0)], [(1, 1), (2, 0)], "added in order"),
    ([PH], [(0, 2, -1, 0)], [(1, 0), (2, 1)], "slop must be >= 0"),
    ([(4, 4, 0, 1.0, 0, 0)], [(0, 2, 0, 0)], [(1, 0), (2, 1)], "bad occur"),
    ([(1, 4, 0, -1.0, 0, 0)], [(0, 2, 0, 0)], [(1, 0), (2, 1)], "Boost must be a positive"),
    ([(1, 7, 0, 1.0, 0, 0)], [(0, 2, 0, 0)], [(1, 0), (2, 1)], "bad clause kind"),
]


@pytest.mark.parametrize("clauses,phrases,terms,msg", INVALID_PHRASES)
def test_invalid_phrases(d, clauses, phrases, terms, msg):
    with pytest.raises(ph.PlanError) as e:
        plan_arrays(d, *_arrays(clauses, phrases, terms))
    assert e.value.rc == INVALID and msg in e.value.msg, e.value.msg


@pytest.mark.parametrize("phrase", [PhraseQuery([1, 2]), PhraseQuery([1]), PhraseQuery([]), PhraseQuery([1, 1], slop=1)])
def test_an_image_without_positions_refuses_phrases(d, phrase):
    with pytest.raises(ph.PlanError) as e:
        plan(d, [bq((0, S), (phrase, S))], positions=False)
    assert e.value.rc == INVALID and "without position data" in e.value.msg
    plan(d, [bq((0, S), (1, S))], positions=False)   # no phrase: no positions needed


def test_unsupported_phrases(d):
    second, again = 1, 2
    cases = [[PhraseQuery([second, second], slop=1)],                                  # "second second"~1: repeat groups
             [bq((PhraseQuery([0, 1, 2, 3, 4]), M), (5, S), (6, S), (7, S), (8, S))],   # 9 term slots
             [bq((PhraseQuery([0, 1, 2, 3, 4, 5]), S), (PhraseQuery([6, 7, 6]), S))],  # 9 slots, phrases only
             [bq(*[(PhraseQuery([]), S)] * 30, (PhraseQuery([0, 1, 2]), S))]]          # 33 clauses with its terms
    for qs in cases:
        with pytest.raises(ph.PlanError) as e:
            plan(d, qs)
        assert e.value.rc == UNSUPPORTED, e.value.msg
    p, _, _ = plan(d, [PhraseQuery([second, again, second])])   # an exact phrase may repeat a term
    assert p.queries[0]["n_term"] == 3
    p, _, _ = plan(d, [bq((PhraseQuery([0, 1, 2, 3]), M), (PhraseQuery([4, 5, 6, 7]), S))])   # 8 slots
    assert p.queries[0]["n_term"] == 8


def test_the_tree_entry_point_rejects_phrase_clauses(d):
    """Without a phrase table a phrase clause is a bad clause kind (nrtgpu_search_tree and every flat entry point)"""
    carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree([bq((PhraseQuery([1, 2]), M), (bq((0, S)), M))],
                                                                         phrase_table=True)
    for args in ((carr, ncl, narr, nn, qarr, nq), (carr, ncl, narr, 0, qarr, nq)):
        with pytest.raises(ph.PlanError) as e:
            th.plan_compiled(d, *args, 10)
        assert e.value.rc == INVALID and "bad clause kind" in e.value.msg
