"""Kernel-level tests of everything after the kNN candidate GEMM: knn_select_kernel, knn_merge_chunk_kernel,
knn_rescore_kernel (score mapping and rank-safety certificate), knn_exact_chunk_kernel + merge_slices_kernel and the
index-time norms, launched through tests/csrc/knn_stage_b_harness.cu and compared with float64 numpy (tests/knn_stage_b.py).

The end-to-end tests cannot see these kernels either: on their corpora the true top-k is always inside the candidate
list, so the page is right because the candidates are right, not because the certificate is. Here
  * the select / merge lists must equal, key for key, the sorted keys of every eligible entry;
  * integer-valued vectors make every float64 sum exact in any order, so re-scored and exactly scored pages must EQUAL
    the reference's docs and float scores;
  * the certificate's decision is probed 2 % of its bound on either side of the k-th exact score, with hand-made lists;
  * on the corpora of tests/knn_adversarial.py the real bf16 candidate stage provably loses every true neighbour: the
    certificate must reject exactly those queries, and the exact fallback must return the brute-force page."""
import numpy as np
import pytest

import knn_adversarial as adv
import knn_stage_b as kh
import oracle
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import GpuIndex, GpuIndexSearcher
from test_gpu_knn import check, knn_run, vec_shard

pytestmark = pytest.mark.gpu

SIMS = (ix.SIM_L2, ix.SIM_DOT, ix.SIM_COSINE, ix.SIM_MIP)
BYTE = kh.BYTE_FLAG
EPS_BF16 = 2.0**-7
INVALID = 1   # NRTGPU_ERR_INVALID


@pytest.fixture(scope="module")
def harness(built):
    return kh.lib()


def assert_lists(cand, cnt, want, what=""):
    for q, w in enumerate(want):
        assert cnt[q] == len(w), (what, q, int(cnt[q]), len(w))
        bad = np.nonzero(cand[q, :len(w)] != w)[0]
        assert len(bad) == 0, (what, q, int(bad[0]), hex(int(cand[q, bad[0]])), hex(int(w[bad[0]])))


def assert_theta(theta, want, kprime, what=""):
    """theta_out is written iff the list is full, with the k'-th score (bit for bit)."""
    for q, w in enumerate(want):
        exp = kh.key_score(w[kprime - 1:kprime])[0] if len(w) == kprime else kh.THETA_UNSET
        assert np.float32(theta[q]).view(np.uint32) == np.float32(exp).view(np.uint32), (what, q, theta[q], exp)


# ---- knn_select_kernel ----

def _pattern(kind, rng, nq, n):
    if kind == "random":
        return rng.standard_normal((nq, n)).astype(np.float32)
    if kind == "descending":   # nothing after the first k' beats the threshold
        return np.repeat(-np.arange(n, dtype=np.float32)[None, :], nq, axis=0)
    if kind == "ascending":    # every block of 256 beats the threshold: the buffer fills and compacts again and again
        return np.repeat(np.arange(n, dtype=np.float32)[None, :], nq, axis=0)
    if kind == "equal":        # ties order by ordinal ascending
        return np.full((nq, n), 0.75, np.float32)
    special = np.array([0.0, -0.0, np.inf, -np.inf, -3.5, 1e-45, -1e-45, 1e-39, 2.0, -1e30, 1.0000001], np.float32)
    return special[rng.integers(0, len(special), (nq, n))]


@pytest.mark.parametrize("kind", ["random", "descending", "ascending", "equal", "special"])
@pytest.mark.parametrize("kprime", [64, 128, 1024, 1028, 3840])
def test_select_equals_sorted_keys(harness, kprime, kind):
    rng = np.random.default_rng(kprime + len(kind))
    S = _pattern(kind, rng, 3, 32768)
    cand, cnt, theta = kh.select(S, kprime)
    want = kh.select_reference(S, kprime)
    assert_lists(cand, cnt, want, kind)
    assert_theta(theta, want, kprime, kind)


@pytest.mark.parametrize("n_chunk", [1, 255, 256, 257, 65533])
def test_select_chunk_sizes_and_base(harness, n_chunk):
    """Chunk tails around the 256-thread step, a row pitch above the chunk and chunk_base != 0."""
    rng = np.random.default_rng(n_chunk)
    S = rng.standard_normal((4, n_chunk + 3)).astype(np.float32)
    for kprime in (64, 3840):
        cand, cnt, theta = kh.select(S, kprime, chunk_base=1_000_000, n_chunk=n_chunk)
        want = kh.select_reference(S[:, :n_chunk], kprime, chunk_base=1_000_000)
        assert_lists(cand, cnt, want)
        assert_theta(theta, want, kprime)


@pytest.mark.parametrize("kprime", [128, 1028, 3840])
def test_select_carries_lists_across_chunks(harness, kprime):
    """Three chained calls equal one call over the concatenation, and both equal the reference."""
    rng = np.random.default_rng(kprime)
    sizes = (5000, 257, 9000)
    S = rng.standard_normal((5, sum(sizes))).astype(np.float32)
    S[1] = np.sort(S[1])           # ascending over the chunks: every chunk replaces the whole list
    want = kh.select_reference(S, kprime)
    one = kh.select(S, kprime)
    assert_lists(one[0], one[1], want, "one call")
    cand = cnt = theta = None
    base = 0
    for n in sizes:
        cand, cnt, theta = kh.select(np.ascontiguousarray(S[:, base:base + n]), kprime, cand, cnt, theta, chunk_base=base)
        base += n
    assert_lists(cand, cnt, want, "chained")
    assert_theta(theta, want, kprime)


@pytest.mark.parametrize("have", ["kprime-1", "kprime"])
def test_select_incoming_list_almost_full_and_full(harness, have):
    kprime, n = 128, 3000
    rng = np.random.default_rng(len(have))
    m = kprime - 1 if have == "kprime-1" else kprime
    inc = np.sort(kh.make_key(rng.standard_normal(m).astype(np.float32) + 1.0, 500_000 + np.arange(m)))[::-1]
    cand0 = np.zeros((2, kprime), np.uint64)
    cand0[:, :m] = inc
    S = rng.standard_normal((2, n)).astype(np.float32)
    S[1] = -50.0   # nothing of this query's chunk enters a full list; one entry completes an almost full one
    cand, cnt, theta = kh.select(S, kprime, cand0, np.full(2, m, np.int32))
    want = kh.select_reference(S, kprime, incoming=[inc, inc])
    assert_lists(cand, cnt, want)
    assert_theta(theta, want, kprime)


def _masks(rng, n_ords, n_docs):
    vec_docs = rng.permutation(n_docs)[:n_ords].astype(np.int32)
    flt = (rng.random(n_docs) < 0.7).astype(np.uint8)
    live = (rng.random(n_docs) < 0.8).astype(np.uint8)
    rows = (rng.random((3, n_docs)) < np.array([[0.5], [0.05], [0.9]])).astype(np.uint8)
    return vec_docs, flt, live, rows


def test_select_filters(harness):
    """Byte filter, deletes and per-query rows (qrow = -1 mixed in) through a permuted vec_docs, chunk_base != 0."""
    rng = np.random.default_rng(5)
    base, n, n_docs, kprime = 700, 6000, 14000, 128
    vec_docs, flt, live, rows = _masks(rng, base + n, n_docs)
    qrow = np.array([0, -1, 1, 2, -1, 0], np.int32)
    S = rng.standard_normal((6, n)).astype(np.float32)
    ords = base + np.arange(n)
    for use in ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1)):
        kw = dict(filter_docs=flt if use[0] else None, live_docs=live if use[1] else None, vec_docs=vec_docs)
        ok = kh.eligible(ords, 6, rows=rows, qrow=qrow if use[2] else None, **kw)
        cand, cnt, theta = kh.select(S, kprime, chunk_base=base, n_docs=n_docs, row_bits=kh.row_bitmaps(rows) if use[2] else None,
                                     qrow=qrow if use[2] else None, **kw)
        want = kh.select_reference(S, kprime, chunk_base=base, ok=ok)
        assert_lists(cand, cnt, want, use)
        assert_theta(theta, want, kprime, use)


@pytest.mark.parametrize("left", [127, 128])
def test_select_filter_leaves_fewer_than_or_exactly_kprime(harness, left):
    """A list that never fills leaves the threshold output untouched; one that fills exactly writes the k'-th score."""
    rng = np.random.default_rng(left)
    n, kprime = 9000, 128
    flt = np.zeros(n, np.uint8)
    flt[rng.choice(n, left, replace=False)] = 1
    S = rng.standard_normal((2, n)).astype(np.float32)
    cand, cnt, theta = kh.select(S, kprime, filter_docs=flt, n_docs=n)
    want = kh.select_reference(S, kprime, ok=kh.eligible(np.arange(n), 2, filter_docs=flt))
    assert all(len(w) == left for w in want)
    assert_lists(cand, cnt, want)
    assert_theta(theta, want, kprime)


def test_harness_refuses_out_of_range_arguments(harness):
    """No test can make a kernel index out of bounds: the harness answers INVALID before it launches."""
    S = np.zeros((1, 10), np.float32)
    with pytest.raises(RuntimeError):
        kh.select(S, 4096 - 255)
    with pytest.raises(RuntimeError):
        kh.select(S, 64, np.zeros((1, 64), np.uint64), np.array([65], np.int32))
    with pytest.raises(RuntimeError):
        kh.select(S, 64, filter_docs=np.ones(5, np.uint8), n_docs=5)
    with pytest.raises(RuntimeError):
        kh.select(S, 64, live_docs=np.ones(20, np.uint8), n_docs=20, vec_docs=np.full(10, 20, np.int32))
    with pytest.raises(RuntimeError):
        kh.select(S, 64, n_docs=10, row_bits=np.zeros((1, 1), np.uint32), qrow=np.array([1], np.int32))
    with pytest.raises(RuntimeError):
        kh.merge_chunk(np.zeros((1, 2048), np.uint64), np.zeros(1, np.int32), np.zeros((1, 2049), np.uint64), np.zeros(1, np.int32))
    Q, D = np.ones((1, 4), np.float32), np.ones((3, 4), np.float32)
    cand = kh.make_key(np.zeros((1, 64), np.float32), np.full((1, 64), 3))
    with pytest.raises(RuntimeError):
        kh.rescore(Q, D, ix.SIM_DOT, cand, np.array([1], np.int32), 10, EPS_BF16, 1.0)
    with pytest.raises(RuntimeError):
        kh.rescore(Q, D, ix.SIM_DOT, cand, np.array([0], np.int32), 65, EPS_BF16, 1.0)
    with pytest.raises(RuntimeError):
        kh.exact(Q, D, ix.SIM_DOT, 10, row_bits=np.ones((1, 1), np.uint32), qrow=np.array([0], np.int32), ord_lists=[[3]])
    with pytest.raises(RuntimeError):
        kh.exact(Q, D, ix.SIM_DOT, 10, qsel=[1])


# ---- knn_merge_chunk_kernel ----

def test_merge_chunk_counts_overflow_and_theta(harness):
    kprime, cc_cap = 1024, 3072
    rng = np.random.default_rng(3)
    haves = [0, kprime - 1, kprime]
    ccs = [0, 1, cc_cap - 1, cc_cap, cc_cap + 5]
    cases = [(h, c) for h in haves for c in ccs]
    nq = len(cases)
    # few distinct scores: the same score occurs in both inputs, and the order falls to the ordinals
    cand = np.zeros((nq, kprime), np.uint64)
    cc = kh.make_key(rng.integers(-4, 5, (nq, cc_cap)).astype(np.float32), 5000 + rng.permuted(np.tile(np.arange(cc_cap), (nq, 1)), axis=1))
    for q, (h, _) in enumerate(cases):
        cand[q, :h] = np.sort(kh.make_key(rng.integers(-4, 5, h).astype(np.float32), rng.permutation(5000)[:h]))[::-1]
    have = np.array([h for h, _ in cases], np.int32)
    ccn = np.array([c for _, c in cases], np.int32)
    for keep in (np.arange(nq), np.nonzero(ccn <= cc_cap)[0]):
        out, cnt, theta, ccn_after, ovf = kh.merge_chunk(cand[keep], have[keep], cc[keep], ccn[keep])
        want = [np.sort(np.concatenate([cand[q, :have[q]], cc[q, :min(ccn[q], cc_cap)]]))[::-1][:kprime] for q in keep]
        assert_lists(out, cnt, want)
        assert_theta(theta, want, kprime)            # written iff the merged list is full
        assert (ccn_after == 0).all()
        assert ovf == int((ccn[keep] > cc_cap).any())   # only a count above the buffer raises the flag


# ---- knn_rescore_kernel: scores ----

def _ints(rng, shape, byte=False):
    lim = 128 if byte else 16
    return rng.integers(-lim, lim, size=shape).astype(np.float32)


def _rescore_want(Q, D, sim, boosts, cand_ords, k, vec_docs, doc_base):
    s = kh.exact_scores(Q, D, sim, boosts)
    out = []
    for q, ords in enumerate(cand_ords):
        docs = ords if vec_docs is None else vec_docs[ords]
        d, sc, n = kh.page_reference(s[q][ords], k, docs=docs)
        out.append((d + doc_base, sc, n))
    return out


@pytest.mark.parametrize("dims", [1, 3, 31, 32, 33, 100, 768])
@pytest.mark.parametrize("sim", [*SIMS, ix.SIM_DOT | BYTE, ix.SIM_L2 | BYTE])
def test_rescore_integer_vectors_equal_reference(harness, sim, dims):
    """Candidate counts 0, 1, k - 1, k and k'; a permuted vec_docs and doc_base; boosts 0.25, 1 and 3.7. At dims 1 and 3
    most scores tie, and the page must order them by doc."""
    rng = np.random.default_rng(dims * 7 + sim)
    k, kprime, n = 10, 64, 200
    D, Q = _ints(rng, (n, dims), sim & BYTE), _ints(rng, (5, dims), sim & BYTE)
    vec_docs = rng.permutation(5 * n)[:n].astype(np.int32)
    boosts = np.array([0.25, 1.0, 3.7, 1.0, 0.25], np.float32)
    counts = np.array([0, 1, k - 1, k, kprime], np.int32)
    ords = [rng.permutation(n)[:c] for c in counts]
    cand = np.zeros((5, kprime), np.uint64)
    for q, o in enumerate(ords):
        cand[q, :len(o)] = kh.make_key(-np.arange(len(o), dtype=np.float32), o)
    docs, scores, cnt, _ = kh.rescore(Q, D, sim, cand, counts, k, EPS_BF16, 1.0, vec_docs=vec_docs, doc_base=1000, boosts=boosts)
    for q, (wd, ws, wn) in enumerate(_rescore_want(Q, D, sim, boosts, ords, k, vec_docs, 1000)):
        assert cnt[q] == wn, q
        assert np.array_equal(scores[q, :wn].view(np.uint32), ws.view(np.uint32)), (q, scores[q, :wn], ws)
        assert np.array_equal(docs[q, :wn], wd), q


@pytest.mark.parametrize("sim", SIMS)
def test_rescore_gaussian_within_one_ulp(harness, sim):
    rng = np.random.default_rng(sim)
    n, dims, k = 128, 100, 128
    D, Q = rng.standard_normal((n, dims)).astype(np.float32), rng.standard_normal((4, dims)).astype(np.float32)
    cand = np.repeat(kh.make_key(-np.arange(n, dtype=np.float32), np.arange(n))[None, :], 4, axis=0)
    docs, scores, cnt, _ = kh.rescore(Q, D, sim, cand, np.full(4, n, np.int32), k, EPS_BF16, 1.0)
    want = kh.exact_scores(Q, D, sim)
    for q in range(4):
        assert cnt[q] == n and sorted(docs[q]) == list(range(n))
        assert (np.abs(scores[q] - want[q][docs[q]]) <= np.spacing(want[q][docs[q]])).all(), q
        assert (np.diff(scores[q]) <= 0).all()


@pytest.mark.parametrize("sim", [*SIMS, ix.SIM_DOT | BYTE])
def test_rescore_edges_equal_oracle(harness, sim):
    """Negative dots (the DOT clamp at 0 with ties by doc, MIP's 1 / (1 - dot) branch), a zero corpus vector and a zero
    query (cosine: NaN -> 0): the kernel, the numpy reference and the oracle agree bit for bit on integer data."""
    rng = np.random.default_rng(40 + sim)
    n, dims = 60, 8
    D, Q = _ints(rng, (n, dims), sim & BYTE), _ints(rng, (4, dims), sim & BYTE)
    D[7] = 0
    D[30:40] = -np.abs(D[30:40]) * np.sign(Q[0] + 0.5)   # dots with query 0 far below -1
    Q[2] = 0
    cand = np.zeros((4, 64), np.uint64)
    cand[:, :n] = kh.make_key(np.zeros(n, np.float32), np.arange(n))
    docs, scores, cnt, _ = kh.rescore(Q, D, sim, cand, np.full(4, n, np.int32), n, EPS_BF16, 1.0)
    wd, ws, wc = oracle.knn_exact(D, sim, Q, n)
    ref = kh.exact_scores(Q, D, sim)
    if (sim & 0xff) == ix.SIM_DOT and not sim & BYTE:
        assert (ref[0][30:40] == 0).all()
    if (sim & 0xff) == ix.SIM_MIP:
        assert (ref[0] < 1).any() and (ref[0] > 1).any()
    for q in range(4):
        rd, rs, _ = kh.page_reference(ref[q], n)
        assert cnt[q] == wc[q] == n
        assert np.array_equal(scores[q].view(np.uint32), ws[q].view(np.uint32)) and np.array_equal(docs[q], wd[q]), q
        assert np.array_equal(rs.view(np.uint32), ws[q].view(np.uint32)) and np.array_equal(rd, wd[q]), q


# ---- knn_rescore_kernel: the certificate's decision ----

def _crossing(sim, dims, qn, dmax, eps, boost, kth, slack):
    """The approximate score th at which the bound on a vector outside the list reaches the k-th exact score (bisection
    on the float64 statement). slack: with the kernel's documented extra room (1 + 1e-3 on eps, 1 + 1e-6 and a float
    round-up on the score), so that a list below it must be accepted."""
    e, f = (eps * (1 + 1e-3), 1 + 2e-6) if slack else (eps, 1.0)
    g = lambda th: kh.score_upper_bound_reference(sim, dims, th, qn, dmax, e, boost) * f - kth
    lo, hi = -1e9, 1e9
    assert g(lo) < 0 < g(hi)
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if g(mid) < 0 else (lo, mid)
    return lo


def _f32_at_most(x):
    f = np.float32(x)
    return f if float(f) <= x else np.nextafter(f, np.float32(-np.inf))


def _f32_at_least(x):
    f = np.float32(x)
    return f if float(f) >= x else np.nextafter(f, np.float32(np.inf))


def _decision_case(sim, boost, eps_kind, q_scale=1.0, seed=0):
    """Two copies of one query over 64 integer vectors, k = 10, k' = 64, every vector a candidate. The weakest
    candidate's approximate score sits 2 % of the bound on the safe side (query 0) and on the unsafe side (query 1)."""
    rng = np.random.default_rng(seed + 10 * sim)
    dims, k, kprime = 32, 10, 64
    lim = 100 if sim & BYTE else 15
    D = rng.integers(0, lim + 1, (kprime, dims)).astype(np.float32)
    q = (rng.integers(1, lim + 1, dims) * q_scale).astype(np.float32)
    Q = np.stack([q, q])
    eps = EPS_BF16 if eps_kind == "bf16" else dims * 2.0**-23
    dmax = 1.7 * float(np.linalg.norm(D.astype(np.float64), axis=1).max())
    qn = float(np.linalg.norm(q.astype(np.float64)))
    boosts = np.full(2, boost, np.float32)
    kth = float(np.sort(kh.exact_scores(Q[:1], D, sim, boosts[:1])[0])[::-1][k - 1])
    unit = kh.approx_unit(sim, qn, dmax, eps)
    th_safe = _f32_at_most(_crossing(sim, dims, qn, dmax, eps, boost, kth, True) - 0.02 * unit)
    th_unsafe = _f32_at_least(_crossing(sim, dims, qn, dmax, eps, boost, kth, False) + 0.02 * unit)
    assert kh.certificate_reference(sim, dims, th_unsafe, qn, dmax, eps, boost, kth) <= 0
    assert kh.certificate_reference(sim, dims, th_safe, qn, dmax, eps, boost, kth) > 0
    cand = np.zeros((2, kprime), np.uint64)
    for i, th in enumerate((th_safe, th_unsafe)):
        approx = np.concatenate([np.float32(th) + np.abs(np.float32(th)) + np.arange(kprime - 1, 0, -1, dtype=np.float32), [th]])
        cand[i] = kh.make_key(approx.astype(np.float32), rng.permutation(kprime))
    return Q, D, cand, k, eps, dmax, boosts


@pytest.mark.parametrize("eps_kind", ["bf16", "fp32"])
@pytest.mark.parametrize("boost", [0.5, 1.0, 2.5])
@pytest.mark.parametrize("sim", [*SIMS, *(s | BYTE for s in SIMS)])
def test_certificate_decision_two_percent_either_side(harness, sim, boost, eps_kind):
    """Soundness: a list whose bound reaches the k-th exact score is ALWAYS rejected. And the certificate is not vacuous:
    2 % of the bound below (with the kernel's documented slack) it accepts. dmax != 1, |q| != 1, both eps_rel values."""
    Q, D, cand, k, eps, dmax, boosts = _decision_case(sim, boost, eps_kind)
    _, _, cnt, unsafe = kh.rescore(Q, D, sim, cand, np.full(2, cand.shape[1], np.int32), k, eps, dmax, boosts=boosts)
    assert list(cnt) == [k, k]
    assert list(unsafe) == [0, 1], unsafe


@pytest.mark.parametrize("sim, q_scale", [(ix.SIM_L2, 1e-3), (ix.SIM_COSINE, 1e-30), (ix.SIM_COSINE, 1e3), (ix.SIM_MIP, 1e-3)])
def test_certificate_decision_small_and_large_queries(harness, sim, q_scale):
    """l2 with |q| about 1e-3 dmax, cosine with a tiny |q| (the bound is relative to |q|, dmax plays no part)."""
    Q, D, cand, k, eps, dmax, boosts = _decision_case(sim, 1.0, "bf16", q_scale=q_scale, seed=1)
    _, _, _, unsafe = kh.rescore(Q, D, sim, cand, np.full(2, cand.shape[1], np.int32), k, eps, dmax, boosts=boosts)
    assert list(unsafe) == [0, 1], unsafe


def test_certificate_decision_special_cases(harness):
    rng = np.random.default_rng(9)
    dims, k, kprime = 32, 10, 64
    D = rng.integers(0, 16, (kprime, dims)).astype(np.float32)
    q = rng.integers(1, 16, dims).astype(np.float32)
    dmax = 1.0001 * float(np.linalg.norm(D.astype(np.float64), axis=1).max())
    full = kh.make_key(np.arange(kprime, 0, -1, dtype=np.float32) - 1e9, np.arange(kprime))   # approximate scores far below
    # a list that is not full has no vector outside it: safe whatever its scores say
    huge = kh.make_key(np.full(kprime, 1e30, np.float32), np.arange(kprime))
    _, _, cnt, unsafe = kh.rescore(q[None], D, ix.SIM_MIP, huge[None], np.array([kprime - 1], np.int32), k, EPS_BF16, dmax)
    assert cnt[0] == k and unsafe[0] == 0
    # the same scores in a full list: rejected; far-below scores: accepted
    _, _, _, unsafe = kh.rescore(np.stack([q, q]), D, ix.SIM_MIP, np.stack([huge, full]), np.full(2, kprime, np.int32), k, EPS_BF16, dmax)
    assert list(unsafe) == [1, 0]
    # boost 0: every score is 0, the bound ties with the k-th score and a tie is not safe
    _, scores, _, unsafe = kh.rescore(q[None], D, ix.SIM_MIP, full[None], np.array([kprime], np.int32), k, EPS_BF16, dmax,
                                      boosts=np.zeros(1, np.float32))
    assert unsafe[0] == 1 and (scores == 0).all()
    # a tie of the bound with the k-th exact score, exactly: DOT scores clamped to 0 on both sides
    neg = -np.abs(D)
    _, scores, _, unsafe = kh.rescore(q[None], neg, ix.SIM_DOT, full[None], np.array([kprime], np.int32), k, EPS_BF16, dmax)
    assert unsafe[0] == 1 and (scores == 0).all()
    # l2 with |q| = 0: the bound has no width, approx = -|d|^2. Safe iff the weakest candidate is strictly farther than the k-th
    z = np.zeros((2, dims), np.float32)
    d2 = np.sort((D.astype(np.float64) ** 2).sum(axis=1))
    lists = np.stack([kh.make_key(np.concatenate([np.zeros(kprime - 1), [-(d2[k - 1] + 64)]]).astype(np.float32), np.arange(kprime)),
                      kh.make_key(np.concatenate([np.zeros(kprime - 1), [-d2[k - 1]]]).astype(np.float32), np.arange(kprime))])
    _, _, _, unsafe = kh.rescore(z, D, ix.SIM_L2, lists, np.full(2, kprime, np.int32), k, EPS_BF16, dmax)
    assert list(unsafe) == [0, 1]


# ---- the certificate as a property of the real candidate stage ----

def _dmax(D):
    """vec_dmax as nrtgpu_index_build computes it."""
    n2 = (D.astype(np.float64) ** 2).sum(axis=1).astype(np.float32)
    return float(np.sqrt(n2.max()) * np.float32(1.0001))


def _assert_safe_pages_exact(a_docs, a_scores, a_cnt, unsafe, wd, ws, k):
    for q in np.nonzero(unsafe == 0)[0]:
        check(a_docs[q:q + 1], a_scores[q:q + 1], a_cnt[q:q + 1], wd[q:q + 1], ws[q:q + 1], np.array([k], np.int32))


@pytest.mark.parametrize("sim", SIMS)
def test_certificate_rejects_lists_that_miss_true_neighbours(harness, sim):
    """knn_gemm_bf16_kernel -> knn_select_kernel -> knn_rescore_kernel on an adversarial corpus: the candidate lists of
    the adversarial queries hold no true neighbour (asserted from the lists), so their re-scored pages are wrong and the
    certificate must reject them; the Gaussian controls stay certified; the exact kernel returns the brute-force page."""
    a = adv.build(sim)
    S = kh.gemm_scores(a.queries, a.corpus, sim)
    cand, cnt, _ = kh.select(S, a.kprime)
    assert (cnt == a.kprime).all()
    for q in range(a.n_adv):
        assert not np.isin(a.neighbours, kh.key_ord(cand[q])).any(), q
    docs, scores, pc, unsafe = kh.rescore(a.queries, a.corpus, sim, cand, cnt, a.k, EPS_BF16, _dmax(a.corpus))
    wd, ws = adv.brute_force(a)
    assert list(unsafe) == [1] * a.n_adv + [0] * (len(a.queries) - a.n_adv), unsafe
    for q in range(a.n_adv):
        assert not np.isin(docs[q], a.neighbours).any() and set(wd[q]) == set(a.neighbours)
    _assert_safe_pages_exact(docs, scores, pc, unsafe, wd, ws, a.k)
    _, _, xd, xs, xc = kh.exact(a.queries, a.corpus, sim, a.k, qsel=np.arange(a.n_adv))
    check(xd, xs, xc, wd[:a.n_adv], ws[:a.n_adv], np.full(a.n_adv, a.k, np.int32))


@pytest.mark.parametrize("sim", [ix.SIM_DOT, ix.SIM_L2])
def test_certificate_rejects_neighbours_dropped_by_the_fused_threshold(harness, sim):
    """The fused schedule by hand: warm chunk through knn_select_kernel, then two fused chunks through the GEMM epilogue
    and knn_merge_chunk_kernel. The decoys raise the threshold in the first fused chunk; the neighbours lie in the second
    and never leave the epilogue."""
    a = adv.build(sim, fused=True)
    n, cc_cap = len(a.corpus), 3072
    S = kh.gemm_scores(a.queries, a.corpus, sim, n_base=0, N=adv.WARM)
    cand, cnt, theta = kh.select(S, a.kprime, theta=np.full(len(a.queries), -np.inf, np.float32))
    for base, size in ((adv.WARM, adv.CHUNK1), (adv.WARM + adv.CHUNK1, n - adv.WARM - adv.CHUNK1)):
        cc, ccn = kh.gemm_fused(a.queries, a.corpus, sim, theta, cc_cap, n_base=base, N=size)
        assert (ccn <= cc_cap).all()
        if base > adv.WARM:
            for q in range(a.n_adv):
                assert not np.isin(a.neighbours, kh.key_ord(cc[q, :ccn[q]])).any(), q
        cand, cnt, theta, _, ovf = kh.merge_chunk(cand, cnt, cc, ccn, theta)
        assert ovf == 0
    for q in range(a.n_adv):
        assert np.isin(kh.key_ord(cand[q]), a.decoys).all(), q
    docs, scores, pc, unsafe = kh.rescore(a.queries, a.corpus, sim, cand, cnt, a.k, EPS_BF16, _dmax(a.corpus))
    wd, ws = adv.brute_force(a)
    assert list(unsafe) == [1] * a.n_adv + [0] * (len(a.queries) - a.n_adv), unsafe
    _assert_safe_pages_exact(docs, scores, pc, unsafe, wd, ws, a.k)
    _, _, xd, xs, xc = kh.exact(a.queries, a.corpus, sim, a.k, qsel=np.arange(a.n_adv))
    check(xd, xs, xc, wd[:a.n_adv], ws[:a.n_adv], np.full(a.n_adv, a.k, np.int32))


@pytest.mark.parametrize("kind", ["gauss", "clustered"])
@pytest.mark.parametrize("sim", SIMS)
def test_certified_pages_equal_brute_force_on_random_corpora(harness, sim, kind):
    """unsafe == 0 implies the page is the brute-force page, on Gaussian data (mostly certified) and on tight clusters
    around the queries (mostly rejected)."""
    rng = np.random.default_rng(70 + sim + len(kind))
    n, dims, nq, k, kp = 6000, 64, 24, 10, 128
    D = rng.standard_normal((n, dims)).astype(np.float32)
    Q = rng.standard_normal((nq, dims)).astype(np.float32)
    if kind == "clustered":
        for q in range(0, nq, 2):
            D[q * 200:q * 200 + 200] = Q[q] * (1 + 0.001 * rng.standard_normal((200, 1))) + 0.01 * rng.standard_normal((200, dims))
    D = D.astype(np.float32)
    cand, cnt, _ = kh.select(kh.gemm_scores(Q, D, sim), kp)
    docs, scores, pc, unsafe = kh.rescore(Q, D, sim, cand, cnt, k, EPS_BF16, _dmax(D))
    s = kh.exact_scores(Q, D, sim)
    pages = [kh.page_reference(s[q], k) for q in range(nq)]
    wd, ws = np.stack([p[0] for p in pages]), np.stack([p[1] for p in pages])
    assert (unsafe == 0).any()
    if kind == "clustered":
        assert (unsafe[0::2] == 1).all()
    _assert_safe_pages_exact(docs, scores, pc, unsafe, wd, ws, k)


# ---- knn_exact_chunk_kernel + merge_slices_kernel ----

def _exact_want(scores_q, entries, ok_q, k, docs_of):
    """(chunk keys [n_chunks][k], chunk counts, page docs, page scores) of one query over the listed ordinals."""
    n_chunks = max(1, -(-len(entries) // kh.EXACT_CHUNK))
    keys, cnt = np.zeros((n_chunks, k), np.uint64), np.zeros(n_chunks, np.int32)
    for c in range(n_chunks):
        e = entries[c * kh.EXACT_CHUNK:(c + 1) * kh.EXACT_CHUNK]
        e = e[ok_q[e]]
        kk = np.sort(kh.make_key(scores_q[e], docs_of[e]))[::-1][:k]
        keys[c, :len(kk)], cnt[c] = kk, len(kk)
    e = entries[ok_q[entries]]
    d, s, _ = kh.page_reference(scores_q[e], k, docs=docs_of[e])
    return keys, cnt, d, s


def _assert_exact(got, want_per_q, doc_base=0):
    keys, cnt, docs, scores, counts = got
    for i, (wk, wc, wd, ws) in enumerate(want_per_q):
        nc = len(wc)
        assert np.array_equal(cnt[i, :nc], wc) and (cnt[i, nc:] == 0).all(), (i, cnt[i], wc)   # eligible vectors, capped at k
        assert np.array_equal(keys[i, :nc], wk), i
        assert counts[i] == len(wd), (i, counts[i], len(wd))
        assert np.array_equal(docs[i, :len(wd)], wd + doc_base), i
        assert np.array_equal(scores[i, :len(wd)].view(np.uint32), ws.view(np.uint32)), i


@pytest.mark.parametrize("k", [1, 10, 1024])
@pytest.mark.parametrize("n", [1, 4095, 4096, 4097, 3 * 4096 + 1])
def test_exact_full_corpus_equals_reference(harness, n, k):
    """Chunk tails on either side of 4096; the best vector at entry 0 and 4095 of a chunk and at n - 1 (equal scores in
    different chunks: doc ascending through the merge); a chunk whose vectors are all filtered between two live ones;
    deletes, boosts, doc_base."""
    rng = np.random.default_rng(n + k)
    sim = SIMS[(n + k) % 4]
    dims = 8
    D, Q = _ints(rng, (n, dims)), _ints(rng, (4, dims))
    Q[0, 0] = 7   # not a zero vector
    best = Q[0] if sim in (ix.SIM_L2, ix.SIM_COSINE) else 15 * np.sign(Q[0])
    for pos in {0, min(4095, n - 1), min(4096, n - 1), n - 1}:
        D[pos] = best
    flt = np.ones(n, np.uint8)
    flt[rng.choice(n, n // 10, replace=False)] = 0
    if n > 2 * 4096:
        flt[4096:8192] = 0
    live = (rng.random(n) < 0.9).astype(np.uint8)
    boosts = np.array([1.0, 0.25, 3.7, 1.0], np.float32)
    for kw in (dict(), dict(filter_docs=flt, live_docs=live, boosts=boosts, doc_base=777)):
        got = kh.exact(Q, D, sim, k, **kw)
        s = kh.exact_scores(Q, D, sim, kw.get("boosts"))
        ok = kh.eligible(np.arange(n), 4, kw.get("filter_docs"), kw.get("live_docs"))
        want = [_exact_want(s[q], np.arange(n), ok[q], k, np.arange(n)) for q in range(4)]
        if kw and n > 2 * 4096:
            assert all(w[1][1] == 0 and w[1][0] > 0 and w[1][2] > 0 for w in want)
        _assert_exact(got, want, kw.get("doc_base", 0))


def test_exact_gather_mode_equals_reference(harness):
    """ords mode: ordinal lists of 0, 1, 4096 and 4097 entries, two queries sharing a row, and a query without a row
    that scores every vector in the same launch; qsel picks the queries out of order."""
    rng = np.random.default_rng(12)
    n, dims, k = 3 * 4096 + 1, 8, 10
    sim = ix.SIM_MIP
    D, Q = _ints(rng, (n, dims)), _ints(rng, (7, dims))
    lists = [np.sort(rng.choice(n, m, replace=False)).astype(np.int32) for m in (0, 1, 4096, 4097)]
    rows = np.zeros((4, n), np.uint8)
    for r, l in enumerate(lists):
        rows[r, l] = 1
    qrow = np.array([3, 0, -1, 2, 1, 3, 0], np.int32)
    qsel = np.array([5, 0, 2, 3, 4, 1], np.int32)
    live = (rng.random(n) < 0.9).astype(np.uint8)
    got = kh.exact(Q, D, sim, k, qsel=qsel, live_docs=live, row_bits=kh.row_bitmaps(rows), qrow=qrow, ord_lists=lists)
    assert got[0].shape[1] == 4
    s = kh.exact_scores(Q, D, sim)
    ok = kh.eligible(np.arange(n), 7, live_docs=live, rows=rows, qrow=qrow)
    want = [_exact_want(s[q], np.arange(n) if qrow[q] < 0 else lists[qrow[q]].astype(np.int64), ok[q], k, np.arange(n)) for q in qsel]
    _assert_exact(got, want)


# ---- index-time preparation ----

@pytest.mark.parametrize("dims", [1, 31, 32, 33, 1001])
def test_prepare_norms_max_and_affine_map(harness, dims):
    rng = np.random.default_rng(dims)
    D = rng.standard_normal((300, dims)).astype(np.float32)
    D[17] = 0
    want = (D.astype(np.float64) ** 2).sum(axis=1)
    for sim in SIMS:
        norm2, mx, ab = kh.prepare(D, sim)
        assert np.array_equal(norm2, want.astype(np.float32))
        assert mx.view(np.uint32) == norm2.max().view(np.uint32)
        if sim == ix.SIM_L2:
            assert np.array_equal(ab, np.stack([np.full(300, 2.0, np.float32), -norm2], axis=1))
        elif sim == ix.SIM_COSINE:
            ref = 1.0 / np.sqrt(np.maximum(norm2.astype(np.float64), 1e-30))
            assert np.isfinite(ab).all() and (ab[:, 1] == 0).all()
            assert (np.abs(ab[:, 0] - ref) <= 3 * 2.0**-23 * ref).all()   # rsqrtf: 2 ulp, and 1e-30f is not 1e-30
        else:
            assert (ab[:, 0] == 1).all() and (ab[:, 1] == 0).all()
    for Z in (np.zeros((5, dims), np.float32), D[:1]):
        norm2, mx, _ = kh.prepare(Z, ix.SIM_DOT)
        assert mx.view(np.uint32) == norm2.max().view(np.uint32)


# ---- through the C ABI ----

ABI_CASES = [(sim, k, False) for sim in SIMS for k in (10, 100)] + [(ix.SIM_DOT, 10, True), (ix.SIM_L2, 10, True)]


@pytest.mark.parametrize("sim, k, fused", ABI_CASES)
def test_knn_search_adversarial_corpora(gpu_ctx, sim, k, fused):
    """GpuIndexSearcher.knn on a real index image: the page equals the oracle's, and exactly the adversarial queries
    took the exact fallback (which also pins vec_dmax: a smaller one would certify them). Then with a byte filter and
    deletes that spare the neighbours and the decoys."""
    a = adv.build(sim, k=k, fused=fused)
    n = len(a.corpus)
    gd, gs, gc, unc = knn_run(gpu_ctx, vec_shard(a.corpus, sim), a.queries, k)
    wd, ws, wc = oracle.knn_exact(a.corpus, sim, a.queries, k)
    check(gd, gs, gc, wd, ws, wc)
    assert unc == a.n_adv, unc
    for q in range(a.n_adv):
        assert set(gd[q]) == set(a.neighbours)
    rng = np.random.default_rng(k)
    flt, live = (rng.random(n) < 0.8).astype(np.uint8), (rng.random(n) < 0.9).astype(np.uint8)
    for m in (flt, live):
        m[a.neighbours] = 1
        m[a.decoys] = 1
    gd, gs, gc, unc = knn_run(gpu_ctx, vec_shard(a.corpus, sim, live_docs=live), a.queries, k, filter_docs=flt)
    wd, ws, wc = oracle.knn_exact(a.corpus, sim, a.queries, k, filter_docs=flt, live_docs=live)
    check(gd, gs, gc, wd, ws, wc)
    assert unc == a.n_adv, unc


@pytest.mark.parametrize("sim", SIMS)
def test_knn_search_zero_query_and_zero_vector(gpu_ctx, sim):
    corpus = ix.synth_vectors(3000, 16)
    queries = ix.synth_vectors(6, 16, seed=ix.SEED_VQUERIES)
    corpus[5] = 0
    queries[1] = 0
    gd, gs, gc, _ = knn_run(gpu_ctx, vec_shard(corpus, sim), queries, 10)
    wd, ws, wc = oracle.knn_exact(corpus, sim, queries, 10)
    check(gd, gs, gc, wd, ws, wc)


def test_knn_search_refuses_bad_boosts_and_empty_batches(gpu_ctx):
    """A kNN boost is a BoostQuery boost: negative, -0, NaN and infinite boosts are refused by the C ABI and raise the text
    path's ValueError in Python; boost 0 is legal (every score 0, docs ascending)."""
    import ctypes as C
    from nrtsearch_b200 import _native
    corpus = ix.synth_vectors(2000, 16)
    queries = ix.synth_vectors(4, 16, seed=ix.SEED_VQUERIES)
    gix = GpuIndex(gpu_ctx, vec_shard(corpus, ix.SIM_COSINE))
    try:
        s = GpuIndexSearcher(gix)
        lib = _native.gpu_lib()
        docs, scores, counts = np.zeros((4, 10), np.int32), np.zeros((4, 10), np.float32), np.zeros(4, np.int32)
        ms = np.zeros(3, np.float32)
        for bad in (-1.0, -0.0, np.nan, np.inf):
            b = np.array([1.0, 1.0, bad, 1.0], np.float32)
            with pytest.raises(ValueError, match="Boost must be a positive number"):
                s.knn(queries, 10, boosts=b)
            with pytest.raises(ValueError, match="Boost must be a positive number"):
                s.knn(queries, 10, boosts=b, filter_queries=[None] * 4)
            rc = lib.nrtgpu_search_knn(gix.handle, queries.ctypes.data, 4, 10, b.ctypes.data, None, C.c_void_p(0),
                                       docs.ctypes.data, scores.ctypes.data, counts.ctypes.data)
            assert rc == INVALID and b"boost" in lib.nrtgpu_last_error()
        for nq in (0, -1):
            assert lib.nrtgpu_search_knn(gix.handle, queries.ctypes.data, nq, 10, None, None, C.c_void_p(0), docs.ctypes.data,
                                         scores.ctypes.data, counts.ctypes.data) == INVALID
            assert lib.nrtgpu_search_knn_timed(gix.handle, queries.ctypes.data, nq, 10, C.c_void_p(0), docs.ctypes.data,
                                               scores.ctypes.data, counts.ctypes.data, ms.ctypes.data) == INVALID
        b = np.array([1.0, 0.0, 2.0, 0.0], np.float32)
        gd, gs, gc = s.knn(queries, 10, boosts=b)
        wd, ws, wc = oracle.knn_exact(corpus, ix.SIM_COSINE, queries, 10, boosts=b)
        check(gd, gs, gc, wd, ws, wc)
        assert list(gd[1]) == list(range(10)) and (gs[1] == 0).all()
    finally:
        gix.close()
