"""CPU proofs of what the GPU tests of the kNN certificate rely on (tests/test_gpu_knn_stage_b.py): the adversarial
corpora of tests/knn_adversarial.py really defeat a bf16 ranking and a sound certificate can still exist; the score
mapping restated in numpy equals the oracle's; the certificate's statement gives hand-computed answers."""
import numpy as np
import pytest

import knn_adversarial as adv
import knn_stage_b as kh
import oracle

SIMS = (kh.SIM_L2, kh.SIM_DOT, kh.SIM_COSINE, kh.SIM_MIP)
EPS_BF16 = 2.0**-7


def bf16_list(a: adv.Adversarial, q: int, n: int = None):
    """(ordinals, approximate scores) of the best k' vectors of corpus[:n] in the bf16 ranking, best first."""
    s = adv.approx_bf16(a.queries[q:q + 1], a.corpus[:n], a.sim)[0]
    order = np.lexsort((np.arange(len(s)), -s))[:a.kprime]
    return order, s[order]


# the layouts the GPU tests use: inside the warm chunk at k = 10 and 100, over the fused chunks for dot and l2
BUILDS = [(sim, k, False) for sim in SIMS for k in (10, 100)] + [(kh.SIM_DOT, 10, True), (kh.SIM_L2, 10, True)]


@pytest.mark.parametrize("sim, k, fused", BUILDS)
def test_builders_defeat_bf16_and_leave_room_for_a_sound_certificate(sim, k, fused):
    a = adv.build(sim, k=k, fused=fused)
    D64 = a.corpus.astype(np.float64)
    dmax = np.linalg.norm(D64, axis=1).max() * 1.0001
    exact = kh.exact_scores(a.queries, a.corpus, sim)
    assert len(a.decoys) > a.kprime
    for q in range(len(a.queries)):
        qn = np.linalg.norm(a.queries[q].astype(np.float64))
        cand, approx = bf16_list(a, q)
        top, _, _ = kh.page_reference(exact[q], k)
        kth = np.sort(exact[q][cand])[::-1][k - 1]
        margin = kh.certificate_reference(sim, adv.DIMS, np.float32(approx[-1]), qn, dmax, EPS_BF16, 1.0, kth)
        if q >= a.n_adv:   # Gaussian control: the bf16 list holds the true page and the certificate accepts it
            assert np.isin(top, cand).all() and margin > 0, (q, margin)
            continue
        assert set(top) == set(a.neighbours), q                              # the exact top-k is exactly the neighbours
        assert not np.isin(a.neighbours, cand).any() and np.isin(cand, a.decoys).all(), q   # the bf16 top-k' has none
        assert margin < 0, (q, margin)                                       # the statement of DESIGN.md 4.3 rejects the list
        half = kh.certificate_reference(sim, adv.DIMS, np.float32(approx[-1]), qn, dmax, EPS_BF16 / 2, 1.0, kth)
        assert half > 0, (q, half)                                           # ... and a bound of 2^-8 would accept it
        # the neighbours' bf16 dot products read between 2^-8 and 2^-7 |q||d| low: a sound bound exists, half of it is not one
        nb = a.corpus[a.neighbours]
        err = (a.queries[q].astype(np.float64) @ nb.astype(np.float64).T
               - kh.bf16_round(a.queries[q]).astype(np.float64) @ kh.bf16_round(nb).astype(np.float64).T)
        rel = err / (qn * np.linalg.norm(nb.astype(np.float64), axis=1))
        assert (rel > 2.0**-8).all() and (rel < 2.0**-7).all(), rel
        if fused:   # after the warm chunk and the decoys' chunk the threshold is above every neighbour's bf16 score
            n1 = adv.WARM + adv.CHUNK1
            assert a.decoys.min() >= adv.WARM and a.decoys.max() < n1 <= a.neighbours.min()
            _, seen = bf16_list(a, q, n1)
            _, warm = bf16_list(a, q, adv.WARM)
            assert adv.approx_bf16(a.queries[q:q + 1], nb, sim).max() < seen[-1] and warm[-1] < seen[-1]


@pytest.mark.parametrize("byte", [False, True])
@pytest.mark.parametrize("sim", SIMS)
def test_map_score_reference_equals_oracle_on_integer_data(sim, byte):
    """Integer vectors: every float64 sum is exact in any order, so the numpy restatement and the oracle's C must agree
    bit for bit, boosts included. Zero vectors (cosine NaN -> 0) and negative dots (DOT clamp, MIP's other branch) are in."""
    rng = np.random.default_rng(sim + 10 * byte)
    lim = 128 if byte else 16
    for dims in (1, 3, 33, 100):
        D = rng.integers(-lim, lim, (300, dims)).astype(np.float32)
        Q = rng.integers(-lim, lim, (6, dims)).astype(np.float32)
        D[7] = 0
        Q[2] = 0
        boosts = np.array([1, 0.25, 3.7, 1, 0.5, 0], np.float32)
        s = sim | (kh.BYTE_FLAG if byte else 0)
        want_d, want_s, want_c = oracle.knn_exact(D, s, Q, 300, boosts=boosts)
        got = kh.exact_scores(Q, D, s, boosts)
        for q in range(len(Q)):
            docs, scores, n = kh.page_reference(got[q], 300)
            assert n == want_c[q] == 300
            assert np.array_equal(scores.view(np.uint32), want_s[q].view(np.uint32)), (dims, q)
            assert np.array_equal(docs, want_d[q]), (dims, q)


E = 2.0**-7
CERT_CASES = [
    # sim, dims, th, |q|, dmax, eps, boost -> the largest score of a vector outside the list, worked by hand
    (kh.SIM_DOT, 8, 10.0, 2.0, 4.0, E, 1.0, (1 + 10.0625) / 2),            # 10 + 2^-7 * 8 = 10.0625
    (kh.SIM_DOT, 8, 10.0, 2.0, 4.0, E, 2.0, 11.0625),
    (kh.SIM_DOT, 8, -3.0, 2.0, 4.0, E, 1.0, 0.0),                          # (1 - 2.9375) / 2 < 0 clamps to 0
    (kh.SIM_MIP, 8, 10.0, 2.0, 4.0, E, 1.0, 11.0625),
    (kh.SIM_MIP, 8, -1.0, 2.0, 4.0, E, 1.0, 1 / 1.9375),                   # -1 + 0.0625 < 0: 1 / (1 + 0.9375)
    (kh.SIM_MIP, 8, -0.0625, 2.0, 4.0, E, 0.5, 0.5),                       # exactly 0: 0 + 1, halved
    (kh.SIM_COSINE, 8, 1.5, 2.0, 99.0, E, 1.0, (1 + 0.7578125) / 2),       # (1.5 + 2^-7 * 2) / 2; dmax plays no part
    (kh.SIM_COSINE, 8, 2.0, 2.0, 99.0, E, 1.0, 1.0),                       # a cosine above 1 clamps to 1
    (kh.SIM_COSINE, 8, -2.5, 2.0, 99.0, E, 3.0, 0.0),
    (kh.SIM_L2, 8, 7.0, 3.0, 4.0, E, 1.0, 1 / (1 + 9 - 7.1875)),           # 7 + 2 * 2^-7 * 12 = 7.1875
    (kh.SIM_L2, 8, 9.0, 3.0, 4.0, E, 1.0, 1.0),                            # a distance below 0 clamps to 0
    (kh.SIM_L2, 8, -1.0, 3.0, 4.0, E, 2.0, 2 / (1 + 9 + 0.8125)),
    (kh.SIM_DOT | kh.BYTE_FLAG, 4, 1000.0, 100.0, 200.0, 4 * 2.0**-23, 1.0, 0.5 + (1000 + 80000 * 2.0**-23) / 131072),
    (kh.SIM_DOT | kh.BYTE_FLAG, 4, -70000.0, 100.0, 200.0, 4 * 2.0**-23, 1.0, 0.0),
    (kh.SIM_DOT | kh.BYTE_FLAG, 4, 0.0, 0.0, 200.0, 4 * 2.0**-23, 2.0, 1.0),
]


@pytest.mark.parametrize("case", CERT_CASES, ids=lambda c: f"sim{c[0]}-th{c[2]}-b{c[6]}")
def test_certificate_reference_hand_computed(case):
    sim, dims, th, qn, dmax, eps, boost, ub = case
    assert kh.score_upper_bound_reference(sim, dims, th, qn, dmax, eps, boost) == pytest.approx(ub, rel=1e-15, abs=0)
    assert kh.certificate_reference(sim, dims, th, qn, dmax, eps, boost, ub + 0.25) == pytest.approx(0.25, rel=1e-12)
    assert kh.certificate_reference(sim, dims, th, qn, dmax, eps, boost, ub) <= 0   # a tie with the bound is not safe
