"""The multi-phrase reference (tests/multi_phrase_reference.py) against the reference project's answers and hand-computed
floats (CPU). The documents of MatchPhrasePrefixQueryTest and MultiMatchPhrasePrefixQueryTest are a tiny shard with
positions; a query's text is split into tokens, every token but the last is looked up in the field's sorted term
dictionary, and the last is expanded as the reference's getPrefixTerms expands it."""
import ctypes as C

import numpy as np
import pytest

import multi_phrase_reference as mpr
import oracle
import phrase_reference as pr
import score_nodes_reference as snr
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, ConstantScoreQuery, DisjunctionMaxQuery, MatchPhrasePrefixQuery,
                                   MultiPhraseQuery, Occur, PhraseQuery, TermQuery)

TEXT1 = ["t1 t2 p1", "t1 t2 p2", "t1 t2 p3", "t1 t2 r1 p1", "t1 t2 r2 p2", "t1 t3 p1", "t1 t3 p2", "t1 t3 p3", "t1 t3 p3",
         "t1 t3 r1 p3", "t1 t3 r2 p4"]
TEXT2 = ["t3 t1 p1", "t3 t1 p2", "t3 t1 p3", "t3 t1 r1 p1", "t3 t1 r2 p2", "t1 t2 p1", "t1 t2 p2", "t1 t2 p3", "t1 t2 p3",
         "t1 t2 r1 p3", "t1 t2 r2 p4"]
VOCAB = sorted({w for t in TEXT1 + TEXT2 for w in t.split()})   # one sorted dictionary per field: term id f * |V| + i


def shard(texts_per_field):
    n_f = len(texts_per_field)
    docs = [[[[f * len(VOCAB) + VOCAB.index(w) for w in texts[d].split()]] for f, texts in enumerate(texts_per_field)]
            for d in range(len(texts_per_field[0]))]
    return pr.shard_from_tokens(docs, np.repeat(np.arange(n_f), len(VOCAB)), n_f)


@pytest.fixture(scope="module")
def one_field():
    sh = shard([TEXT1])
    return sh, oracle.OracleIndex(sh)


@pytest.fixture(scope="module")
def two_fields():
    sh = shard([TEXT1, TEXT2])
    return sh, oracle.OracleIndex(sh)


def phrase_prefix(text, slop=0, max_expansions=0, field=0):
    """createQueryFromTokenStream + the adaptor's expansion: the MatchPhrasePrefixQuery of `text` on `field`"""
    toks = text.split()
    if not toks:
        return MultiPhraseQuery([])
    dictionary = [w.encode() for w in VOCAB]
    exp = mpr.expand_prefix([dictionary], toks[-1].encode(), max_expansions)
    base = field * len(VOCAB)
    return MatchPhrasePrefixQuery([[base + VOCAB.index(w)] for w in toks[:-1]], [base + dictionary.index(e) for e in exp], slop)


def hits(sh, oix, q):
    docs, _, counts, total, _ = mpr.search(sh, [q], 20, oix=oix)
    return sorted(docs[0, :counts[0]].tolist())


@pytest.mark.parametrize("text,slop,max_exp,want", [
    ("t1 t2 p", 0, 0, [0, 1, 2]),                              # testTextPhrasePrefixQuery
    ("t1 t2 p", 1, 0, [0, 1, 2, 3, 4]),                        # testTextSlop
    ("t1 r", 1, 0, [3, 4, 9, 10]),
    ("t1 t2 p", 0, 1, [0]),                                    # testTextMaxExpansions
    ("t1 t2 r", 0, 1, [3]),
    ("t1 t3 r", 0, 1, [9]),
    ("t1 t", 0, 1, []),
    ("p", 0, 0, list(range(11))),                              # testTextPrefixOnly
    ("r", 0, 0, [3, 4, 9, 10]),
    ("", 0, 0, []),                                            # testTextNoQueryTerms
    ("t1 t2 x", 0, 0, []),                                     # an empty expansion after tokens
])
def test_match_phrase_prefix_query_test(one_field, text, slop, max_exp, want):
    sh, oix = one_field
    assert hits(sh, oix, phrase_prefix(text, slop, max_exp)) == want


@pytest.mark.parametrize("text,slop,max_exp,fields,want", [
    ("t1 t2 p", 0, 0, [0], [0, 1, 2]),                         # testMultiMatchPhrasePrefix
    ("t1 t2 p", 0, 0, [1], [5, 6, 7, 8]),
    ("t1 t2 p", 0, 0, [0, 1], [0, 1, 2, 5, 6, 7, 8]),
    ("t1 t3 p", 1, 0, [0, 1], [5, 6, 7, 8, 9, 10]),            # testSlop
    ("t1 t3 p", 2, 0, [0, 1], list(range(11))),
    ("t1 t2 p", 0, 1, [0, 1], [0, 5]),                         # testMaxExpansions
])
def test_multi_match_phrase_prefix_query_test(two_fields, text, slop, max_exp, fields, want):
    sh, oix = two_fields
    q = DisjunctionMaxQuery([phrase_prefix(text, slop, max_exp, f) for f in fields], 0.0)
    assert hits(sh, oix, q) == want


def bm25(sh, weight, freq, doc, f=0):
    fld = sh.fields[f]
    cache = oracle.bm25_cache(fld.k1, fld.b, float(oracle.lib().orc_bm25_avgdl(fld.sum_total_term_freq, fld.doc_count)))
    return np.float32(oracle.lib().orc_bm25_score(np.float32(weight), float(freq), int(fld.norms[doc]), cache.ctypes.data_as(C.POINTER(C.c_float))))


def idf(sh, t):
    return float(oracle.bm25_idf(int(sh.term_df[t]), sh.fields[0].doc_count))


def test_one_token_prefix_is_the_sum_of_its_terms(one_field):
    sh, oix = one_field
    ids = [VOCAB.index(w) for w in ("p1", "p2", "p3", "p4")]
    docs, scores, counts, _, _ = mpr.search(sh, [BoostQuery(MatchPhrasePrefixQuery([], ids), 1.5)], 20, oix=oix)
    got = dict(zip(docs[0, :counts[0]].tolist(), scores[0, :counts[0]].tolist()))
    assert sorted(got) == list(range(11))
    for d in range(11):
        s = 0.0
        for t in ids:   # each doc holds one p term once
            if VOCAB[t] in TEXT1[d].split():
                s += float(bm25(sh, np.float32(1.5) * np.float32(idf(sh, t)), 1, d))
        assert got[d] == np.float32(s)


def test_one_alternative_is_that_term(one_field):
    sh, oix = one_field
    t = VOCAB.index("r1")
    a = mpr.search(sh, [MatchPhrasePrefixQuery([], [t])], 20, oix=oix)
    b = mpr.search(sh, [TermQuery(t)], 20, oix=oix)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_a_term_with_df_0_adds_no_idf(one_field):
    sh, oix = one_field
    sh2 = shard([TEXT1])
    sh2.term_df = sh2.term_df.copy()
    t1, t2, p1, p2 = (VOCAB.index(w) for w in ("t1", "t2", "p1", "p2"))
    absent = VOCAB.index("r2")
    sh2.term_df[absent] = 0   # as if the term were gone from the reader
    q = MultiPhraseQuery([[t1], [t2], [p1, absent]])
    docs, scores, counts, _, _ = mpr.search(sh2, [q], 20)
    got = dict(zip(docs[0, :counts[0]].tolist(), scores[0, :counts[0]].tolist()))
    assert sorted(got) == [0, 4]   # df only weighs: doc 4 still matches through r2's postings
    w = np.float32(idf(sh2, t1) + idf(sh2, t2) + idf(sh2, p1))
    assert got[0] == bm25(sh2, w, 1, 0) and got[4] == bm25(sh2, w, 1, 4)
    sh2.term_df[:] = 0   # no term of the phrase has df > 0: nothing matches
    assert mpr.search(sh2, [q], 20)[2][0] == 0


def test_duplicate_positions_in_a_doc_count_each_lead():
    # doc 0: "a b" with the synonym c stacked on a (same position); the union [a, c] holds position 0 twice, so the exact
    # matcher counts two matches of "[a c] b"
    a, b, c = 0, 1, 2
    sh = pr.shard_from_token_arrays(1, [0, 0, 0], 1, [0, 0, 0], [a, c, b], [0, 0, 1])
    q = MultiPhraseQuery([[a, c], [b]])
    docs, scores, counts, _, _ = mpr.search(sh, [q], 5)
    w = np.float32(sum(float(oracle.bm25_idf(1, 1)) for _ in range(3)))
    assert counts[0] == 1 and scores[0, 0] == bm25(sh, w, 2, 0)
    assert pr.exact_freq([[0, 0], [1]], [0, 1]) == 2


def test_sloppy_multi_phrase(one_field):
    sh, oix = one_field
    t1, t2 = VOCAB.index("t1"), VOCAB.index("t2")
    ps = [VOCAB.index(w) for w in ("p1", "p2")]
    docs, scores, counts, _, _ = mpr.search(sh, [MultiPhraseQuery([[t1], [t2], ps], slop=1)], 20, oix=oix)
    assert docs[0, :counts[0]].tolist() == [0, 1, 3, 4]
    w = np.float32(idf(sh, t1) + idf(sh, t2) + idf(sh, ps[0]) + idf(sh, ps[1]))
    got = dict(zip(docs[0, :counts[0]].tolist(), scores[0, :counts[0]].tolist()))
    assert got[0] == bm25(sh, w, 1, 0)
    assert got[3] == bm25(sh, w, np.float32(1) / np.float32(2), 3)   # "t1 t2 r1 p1": matchLength 1


def test_one_term_per_position_is_the_phrase(one_field):
    sh, oix = one_field
    rng = np.random.default_rng(5)
    for _ in range(40):
        n = int(rng.integers(2, 4))
        terms = [int(t) for t in rng.integers(0, len(VOCAB), n)]
        slop = int(rng.integers(0, 3))
        if slop and len(set(terms)) < n:
            continue
        boost = float(rng.choice([1.0, 0.5, 3.0]))
        a = mpr.search(sh, [BoostQuery(MultiPhraseQuery([[t] for t in terms], slop=slop), boost)], 11, oix=oix)
        b = pr.search(sh, [BoostQuery(PhraseQuery(terms, slop=slop), boost)], 11, oix=oix)
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


def test_generated_trees(two_fields):
    """a few hundred random trees of terms, phrases, multi-phrases, dismaxes and constant-score nodes run through the
    reference (the generator the GPU test checks the device with): pages are ordered and most trees match"""
    sh, oix = two_fields
    rng = np.random.default_rng(11)
    V = len(VOCAB)
    dictionary = [w.encode() for w in VOCAB]

    def leaf():
        f = int(rng.integers(0, 2))
        r = rng.random()
        if r < 0.3:
            return TermQuery(f * V + int(rng.integers(0, V)))
        if r < 0.5:
            return PhraseQuery([f * V + int(t) for t in rng.integers(0, V, 2)])
        toks = [VOCAB[int(i)] for i in rng.integers(0, V, int(rng.integers(1, 3)))]
        text = " ".join(toks[:-1] + [toks[-1][:int(rng.integers(1, 3))]])
        return phrase_prefix(text, int(rng.integers(0, 2)) if rng.random() < 0.3 else 0, int(rng.integers(0, 4)), f)

    def node(depth):
        r = rng.random()
        kids = [leaf() if depth >= 2 or rng.random() < 0.6 else node(depth + 1) for _ in range(int(rng.integers(1, 4)))]
        if r < 0.3:
            return DisjunctionMaxQuery(kids, float(rng.choice([0.0, 0.3])))
        if r < 0.4:
            return ConstantScoreQuery(kids[0])
        b = BooleanQuery()
        for k in kids:
            b.add(BoostQuery(k, float(rng.choice([1.0, 2.0]))), Occur(int(rng.choice([0, 0, 1, 2, 3]))))
        return b

    n_checked = 0
    for _ in range(300):
        q = node(0)
        docs, scores, counts, total, _ = mpr.search(sh, [q], 11, oix=oix)
        n_checked += int(total[0] > 0)
        assert counts[0] == min(11, total[0])
        assert np.all(np.diff(scores[0, :counts[0]].astype(np.float64)) <= 0)
    assert n_checked > 100


def test_a_repeated_term_counts_its_idf_each_time(one_field):
    """'t1 t' expands the prefix to t1, t2, t3, so t1 stands at both positions: MultiPhraseQuery.createWeight adds t1's
    statistics once per occurrence, as PhraseQuery does, and the union of [t1 t2 t3] holds t1's positions too"""
    sh, oix = one_field
    t1, t2, t3 = (VOCAB.index(w) for w in ("t1", "t2", "t3"))
    q = MatchPhrasePrefixQuery([[t1]], [t1, t2, t3])
    docs, scores, counts, _, _ = mpr.search(sh, [q], 20, oix=oix)
    assert sorted(docs[0, :counts[0]].tolist()) == list(range(11))   # "t1 t2" or "t1 t3" starts every doc
    w = np.float32(idf(sh, t1) + idf(sh, t1) + idf(sh, t2) + idf(sh, t3))
    got = dict(zip(docs[0, :counts[0]].tolist(), scores[0, :counts[0]].tolist()))
    assert all(got[d] == bm25(sh, w, 1, d) for d in range(11))
    p = mpr.search(sh, [PhraseQuery([t1, t1])], 20, oix=oix)   # a repeat at one position of each: PhraseQuery's weight too
    m = mpr.search(sh, [MultiPhraseQuery([[t1], [t1]])], 20, oix=oix)
    for x, y in zip(p, m):
        assert np.array_equal(x, y)
