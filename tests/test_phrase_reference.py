"""The phrase reference (tests/phrase_reference.py) pinned to the answers of the reference's own QueryTest on its addDocs.txt
corpus, to hand-derived phrase freqs, and its whole-shard exact matcher to the step-by-step one."""
import numpy as np
import pytest

import oracle
import phrase_reference as pr
from nrtsearch_b200.search import BooleanQuery, MatchAllDocsQuery, Occur, PhraseQuery

FIRST, VENDOR, AGAIN, SECOND = 0, 1, 2, 3


@pytest.fixture(scope="module")
def vendors(built):
    """addDocs.txt's vendor_name: doc_id 1 = ["first vendor", "first again"], doc_id 2 = ["second vendor", "second again"]
    (shard docs 0 and 1), one text field, position increment gap 100"""
    docs = [[[[FIRST, VENDOR], [FIRST, AGAIN]]], [[[SECOND, VENDOR], [SECOND, AGAIN]]]]
    return pr.shard_from_tokens(docs, [0, 0, 0, 0], 1)


def hits(sh, q, k=10):
    d, s, c, t, _ = pr.search(sh, [q], k)
    return d[0, :c[0]].tolist(), s[0, :c[0]], int(t[0])


def test_positions_follow_the_gap(vendors):
    # doc 1: second 0, vendor 1, second 102, again 103
    leaves = pr.PhraseLeaves(vendors, oracle.OracleIndex(vendors), None, None)
    got = {}
    for t in range(4):
        for p, d in zip(*leaves.term_postings(t)):
            if d == 1:
                got[t] = leaves.positions(p)
    assert got == {SECOND: [0, 102], VENDOR: [1], AGAIN: [103]}
    assert vendors.fields[0].sum_total_term_freq == 8 and vendors.fields[0].doc_count == 2


def test_query_test_exact_phrases(vendors):
    # QueryTest.java:192-288: a phrase at the root, as MUST, and as MUST_NOT beside a match-all FILTER
    assert hits(vendors, PhraseQuery([SECOND, AGAIN]))[0] == [1]
    assert hits(vendors, BooleanQuery().add(PhraseQuery([FIRST, AGAIN]), Occur.MUST))[0] == [0]
    q = BooleanQuery().add(PhraseQuery([FIRST, AGAIN]), Occur.MUST_NOT).add(MatchAllDocsQuery(), Occur.FILTER)
    assert hits(vendors, q)[0] == [1]
    assert hits(vendors, PhraseQuery([SECOND, SECOND]))[2] == 0   # QueryTest.java:762-780: split by the gap


def test_query_test_sloppy_phrase_score(vendors):
    # QueryTest.java:738-760 and the explain of :977-1018: "second again"~1 hits doc_id 2 with 0.3979403, phraseFreq=1.0
    docs, scores, total = hits(vendors, PhraseQuery([SECOND, AGAIN], slop=1))
    assert docs == [1] and total == 1
    assert scores[0] == np.float32(0.3979403)
    idf = np.float32(float(oracle.bm25_idf(1, 2)) + float(oracle.bm25_idf(2, 2)))
    assert idf == np.float32(0.87546873)


def test_overlapping_repeats_and_stacked_positions():
    assert pr.exact_freq([[0, 1, 2], [0, 1, 2]], [0, 1]) == 2          # "a a" in "a a a"
    assert pr.exact_freq([[0, 1, 2], [0, 1, 2], [0, 1, 2]], [0, 1, 2]) == 1
    assert pr.exact_freq([[5], [5], [6]], [0, 0, 1]) == 1              # two terms stacked at query position 0
    assert pr.exact_freq([[3, 3], [4]], [0, 1]) == 2                   # the lead's stacked occurrences count each
    assert pr.exact_freq([[4], [3, 3]], [0, 1]) == 0
    assert pr.exact_freq([[0, 7], [1, 9]], [0, 1], first_only=True) == 1


def test_sloppy_match_lengths_sum_in_float():
    # "a b"~2 over a@0 b@1 (length 0), a@10 b@12 (length 1), a@20 b@23 (length 2)
    f = pr.sloppy_freq([[0, 10, 20], [1, 12, 23]], [0, 1], 2)
    want = np.float32(np.float32(np.float32(1) + np.float32(1) / np.float32(2)) + np.float32(1) / np.float32(3))
    assert f.view(np.uint32) == want.view(np.uint32)
    # the reversed pair: b before a costs 2 more (length 2 at distance 1)
    assert pr.sloppy_freq([[1], [0]], [0, 1], 1) == 0
    assert pr.sloppy_freq([[1], [0]], [0, 1], 2) == np.float32(1) / np.float32(3)


def test_slop_at_the_match_length_and_one_less():
    # "vendor again" across the gap of doc_id 2: vendor@1, again@103 -> match length 101
    tp = [[1], [103]]
    assert pr.sloppy_freq(tp, [0, 1], 101) == np.float32(1) / np.float32(102)
    assert pr.sloppy_freq(tp, [0, 1], 100) == 0
    # "vendor second": second@0 before vendor@1 costs 2, second@102 after the gap 100; the shorter one is the match
    assert pr.sloppy_freq([[1], [0, 102]], [0, 1], 2) == np.float32(1) / np.float32(3)
    assert pr.sloppy_freq([[1], [0, 102]], [0, 1], 1) == 0
    # inside one value "second vendor" is exact; the phrase split by the gap is not
    assert pr.exact_freq([[0, 102], [1]], [0, 1]) == 1 and pr.exact_freq([[1], [0, 102]], [0, 1]) == 0


def test_whole_shard_exact_matcher_equals_the_step_by_step_one(built):
    rng = np.random.default_rng(5)
    docs = [[[list(rng.integers(0, 4, rng.integers(1, 12))) for _ in range(rng.integers(1, 3))]] for _ in range(300)]
    sh = pr.shard_from_tokens(docs, [0] * 4, 1, gap=3)
    leaves = pr.PhraseLeaves(sh, oracle.OracleIndex(sh), None, None)
    for terms, offs in [([0, 1], [0, 1]), ([2, 2], [0, 1]), ([1, 0, 1], [0, 1, 2]), ([3, 0], [0, 2]), ([0, 1, 2, 3], [0, 1, 2, 3])]:
        lists = [leaves.term_postings(t) for t in terms]
        cand = lists[0][1]
        for _, d in lists[1:]:
            cand = np.intersect1d(cand, d)
        fast = pr.exact_freqs(sh, leaves.pstart, lists, offs, cand)
        idx = [p[np.searchsorted(d, cand)] for p, d in lists]
        slow = [pr.exact_freq([leaves.positions(idx[i][k]) for i in range(len(terms))], offs) for k in range(len(cand))]
        assert np.array_equal(fast, np.array(slow, np.float32)), (terms, offs)
        assert (fast > 0).any()
