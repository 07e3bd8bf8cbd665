"""The numpy restatement of the top-k kernels (tests/topk_reference.py), which tests/test_gpu_topk_merge.py holds the
kernels to, checked without a GPU: hand-typed answers, the RRF known answers, and random inputs (up to the 4096-key
shapes of the blends) against the C oracle's merge_topk, blend_rrf, blend_scores and rescore_combine."""
import numpy as np
import pytest

import oracle
import topk_reference as ref

SPECIAL = np.array([np.inf, 3.4028235e38, 2.5, 1.0, 1e-40, 1e-45, 0.0, -1e-45, -1.0, -3.4028235e38], np.float32)


def test_key_order_is_pair_order():
    rng = np.random.default_rng(5)
    doc_base = 1 << 20
    scores = np.concatenate([np.repeat(SPECIAL, 8), rng.choice(SPECIAL, 400)]).astype(np.float32)
    docs = rng.choice(np.concatenate([np.arange(300), ref.INT32_MAX - doc_base - np.arange(300)]), len(scores), replace=False)
    keys = ref.make_keys(scores, docs)
    assert len(np.unique(keys)) == len(keys)
    by_key = np.argsort(keys)[::-1]
    assert np.array_equal(by_key, ref.order(scores, docs))
    assert ref.make_keys([1.0], [0])[0] == np.uint64((0xBF800000 << 32) | 0xFFFFFFFF)
    assert ref.make_keys([-1.0], [ref.INT32_MAX])[0] == np.uint64((0x407FFFFF << 32) | 0x80000000)


def test_merge_slices_by_hand():
    # two lists of top_k 3 (the second holds 2 keys); theta = the pair (2.0, 8): (2.0, 9) and below are dropped
    s = np.array([[5.0, 2.0, 1.0], [2.0, 2.0, 0.0]], np.float32)
    d = np.array([[4, 9, 1], [8, 3, 0]], np.int32)
    pd, ps = ref.merge_slices_page(s, d, [3, 2], 3, doc_base=100)
    assert pd.tolist() == [104, 103, 108] and ps.tolist() == [5.0, 2.0, 2.0]
    pd, ps = ref.merge_slices_page(s, d, [3, 2], 10, doc_base=0, theta=(2.0, 8))
    assert pd.tolist() == [4, 3, 8] and ps.tolist() == [5.0, 2.0, 2.0]
    pd, _ = ref.merge_slices_page(s, d, [3, 2], 3, theta=(5.0, 3))
    assert pd.tolist() == []
    # queries: (pruned, terminated in, total, known) with terminate_after 10
    term, total, flags = ref.merge_slices_flags(total_hits=[5, 11, 11, 3], pruned=[0, 0, 1, 1], terminated=[0, 0, 0, 1],
                                                terminate_after=10, known_hits=[9, 9, 20, 2], nq=4)
    assert term.tolist() == [0, 1, 1, 1] and total.tolist() == [5, 11, 20, 3] and flags.tolist() == [0, 3, 3, 3]
    term, total, flags = ref.merge_slices_flags(nq=2)
    assert term is None and total.tolist() == [0, 0] and flags.tolist() == [0, 0]


def test_merge_pairs_by_hand():
    docs = np.array([[[1, 2]], [[0, 5]], [[7, 0]]], np.int32)
    scores = np.array([[[3.0, 1.0]], [[3.0, 2.0]], [[1.0, 0.0]]], np.float32)
    totals = np.full((3, 1), 2**31 - 1, np.int64)
    d, s, c, t, f = ref.merge_pairs(docs, scores, [[2], [2], [1]], 4, totals, [[1], [2], [4]])
    assert d.tolist() == [[0, 1, 5, 2]] and s.tolist() == [[3.0, 3.0, 2.0, 1.0]] and c.tolist() == [4]
    assert t.tolist() == [3 * (2**31 - 1)] and f.tolist() == [7]
    d, s, c, _, _ = ref.merge_pairs(docs, scores, [[0], [1], [0]], 3)
    assert d.tolist() == [[0, 0, 0]] and s.tolist() == [[3.0, 0.0, 0.0]] and c.tolist() == [1]


def test_flush_by_hand():
    s = np.array([4.0, 9.0, 4.0, 1.0], np.float32)
    d = np.array([2, 7, 1, 3], np.int32)
    kth = int(ref.make_keys([4.0], [2])[0])
    pd, ps, n, g, t = ref.flush(s, d, 4, 4, 3, 1, 0, 0)
    assert pd.tolist() == [7, 1, 2] and ps.tolist() == [9.0, 4.0, 4.0] and n == 3 and g == kth - 1 and t == kth - 1
    pd, _, n, g, t = ref.flush(s, d, 4, 4, 3, 0, kth + 5, 0)   # a higher published threshold stays
    assert n == 3 and g == kth + 5 and t == kth + 5
    pd, _, n, g, t = ref.flush(s, d, 2, 4, 3, 0, 17, 20)       # fewer than top_k: nothing is published
    assert pd.tolist() == [7, 2] and n == 2 and g == 17 and t == 20
    pd, _, n, _, _ = ref.flush(s, d, 9, 2, 2, 0, 0, 0)         # a count above cap reads cap keys
    assert pd.tolist() == [7, 2] and n == 2


def test_rrf_known_answers():
    # MultiRetrieverSearchTest.java:410-437: 1/(60+rank) sums (the known answer of test_gpu_hybrid.py)
    d, s, t = ref.blend(0, np.array([[7, 3, 5], [3, 9, 7]]), [3, 3], [1.0, 1.0], 10)
    f = np.float32
    want = {7: f(1) / f(61) + f(1) / f(63), 3: f(1) / f(62) + f(1) / f(61), 5: f(1) / f(63), 9: f(1) / f(62)}
    assert t == 4 and sorted(d.tolist()) == [3, 5, 7, 9]
    assert [want[int(x)] for x in d] == s.tolist() and list(s) == sorted(s, reverse=True)
    # rank_constant <= 0 selects 60
    assert np.array_equal(ref.blend(0, np.array([[7, 3]]), [2], [1.0], 5, rank_constant=0)[1], np.float32([1 / 61, 1 / 62]))


def test_score_blends_by_hand():
    docs = np.array([[4, 2, 6], [2, 4, 6], [6, 9, 9]])
    sc = np.array([[3.0, 2.0, 1.0], [4.0, 1.0, 0.5], [8.0, 1.0, 1.0]], np.float32)
    b = [1.0, 0.5, 0.25]
    d, s, t = ref.blend(1, docs, [3, 3, 1], b, 5, scores=sc)   # MAX
    assert t == 3 and d.tolist() == [4, 2, 6] and s.tolist() == [3.0, 2.0, 2.0]
    d, s, t = ref.blend(2, docs, [3, 3, 1], b, 5, scores=sc)   # SUM
    assert d.tolist() == [2, 4, 6] and s.tolist() == [4.0, 3.5, 3.25]
    d, s, t = ref.blend(3, docs, [3, 3, 1], b, 5, scores=sc)   # running AVG: doc 6 is ((1 + 0.25) / 2 * 2 + 2) / 3
    assert d.tolist() == [2, 4, 6] and s.tolist() == [2.0, 1.75, np.float32(np.float32(np.float32(1.25) / 2 * 2 + 2) / 3)]


def _lists(rng, n_lists, nq, k, n_scores):
    """pages [n_lists, nq, k] ordered best first, docs distinct per query across the lists, scores with many ties"""
    docs = np.stack([rng.permutation(n_lists * k * 4)[:n_lists * k].reshape(n_lists, k) for _ in range(nq)], axis=1)
    scores = rng.choice(np.linspace(-4, 4, n_scores).astype(np.float32), (n_lists, nq, k))
    for l in range(n_lists):
        for q in range(nq):
            o = ref.order(scores[l, q], docs[l, q])
            docs[l, q], scores[l, q] = docs[l, q][o], scores[l, q][o]
    counts = rng.integers(0, k + 1, (n_lists, nq))
    counts[:, 0] = k
    return docs.astype(np.int32), scores.astype(np.float32), counts.astype(np.int32)


@pytest.mark.parametrize("n_lists,k", [(1, 1), (3, 40), (8, 1024), (9, 1023), (64, 40)])
def test_merge_pairs_matches_oracle(built, n_lists, k):
    rng = np.random.default_rng(n_lists * 1000 + k)
    docs, scores, counts = _lists(rng, n_lists, 6, k, 9)
    d, s, c, _, _ = ref.merge_pairs(docs, scores, counts, k)
    wd, ws, wc = oracle.merge_topk(docs, scores, counts, k)
    assert np.array_equal(c, wc)
    for q in range(6):
        assert np.array_equal(d[q, :c[q]], wd[q, :c[q]]) and np.array_equal(s[q, :c[q]].view(np.uint32), ws[q, :c[q]].view(np.uint32))
        assert not d[q, c[q]:].any() and not s[q, c[q]:].view(np.uint32).any()
    # merge_slices_page is the same merge of a query's lists (doc_base 0, no threshold)
    for q in range(6):
        pd, ps = ref.merge_slices_page(scores[:, q], docs[:, q], counts[:, q], k)
        assert np.array_equal(pd, d[q, :c[q]]) and np.array_equal(ps, s[q, :c[q]])


@pytest.mark.parametrize("R,top_in", [(1, 4096), (4, 1024), (64, 64), (3, 100)])
def test_blends_match_oracle(built, R, top_in):
    rng = np.random.default_rng(R * 7 + top_in)
    for heads in (top_in, R * top_in):   # every doc in every retriever; all docs distinct
        for trial in range(2):
            docs = np.stack([rng.permutation(heads)[:top_in] if heads == top_in else np.arange(r * top_in, (r + 1) * top_in)
                             for r in range(R)]).astype(np.int32)
            counts = np.full(R, top_in, np.int32) if trial == 0 else rng.integers(0, top_in + 1, R).astype(np.int32)
            boosts = rng.choice(np.float32([1.0, 0.5, 2.0, 0.7]), R).astype(np.float32)
            scores = np.sort(rng.choice(np.linspace(0, 3, 50).astype(np.float32), (R, top_in)), axis=1)[:, ::-1].copy()
            for top_out in (1, heads, heads + 5):
                d, s, t = ref.blend(0, docs, counts, boosts, top_out, rank_constant=7 if trial else 0)
                wd, ws, wt = oracle.blend_rrf(docs, counts, boosts, 7 if trial else 0, top_out)
                assert t == wt and np.array_equal(d, wd) and np.array_equal(s.view(np.uint32), ws.view(np.uint32))
                for mode in (1, 2, 3):
                    d, s, t = ref.blend(mode, docs, counts, boosts, top_out, scores=scores)
                    wd, ws, wt = oracle.blend_scores(mode, docs, scores, counts, boosts, top_out)
                    assert t == wt and np.array_equal(d, wd) and np.array_equal(s.view(np.uint32), ws.view(np.uint32)), mode


@pytest.mark.parametrize("n", [1, 100, 4096])
def test_rescore_combine_matches_oracle(built, n):
    rng = np.random.default_rng(n)
    docs = rng.permutation(n * 3)[:n].astype(np.int32)
    scores = np.sort(rng.choice(np.linspace(0, 5, 40).astype(np.float32), n))[::-1].copy()
    m = (rng.random(n) < 0.5).astype(np.uint8)
    s2 = rng.choice(np.linspace(0, 2, 30).astype(np.float32), n)
    for qw, rw in ((1.0, 2.0), (0.3, 1.7)):
        d, s = ref.rescore_combine(docs, scores, m, s2, qw, rw)
        wd, ws = oracle.rescore_combine(docs, scores, m, s2, qw, rw)
        assert np.array_equal(d, wd) and np.array_equal(s.view(np.uint32), ws.view(np.uint32))
    c = n // 2
    d, s = ref.rescore_combine(docs, scores, m, s2, 1.0, 2.0, count=c)
    wd, ws = oracle.rescore_combine(docs[:c], scores[:c], m[:c], s2[:c], 1.0, 2.0)
    assert np.array_equal(d[:c], wd) and np.array_equal(s[:c], ws) and np.array_equal(d[c:], docs[c:])
