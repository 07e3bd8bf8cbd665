"""Kernel-level tests of the kNN candidate stage: tc::knn_gemm_bf16_kernel (TMA + wgmma, unfused and fused epilogue) and
knn_dot_tile_kernel (fp32 SIMT), launched directly through tests/csrc/knn_harness.cu and compared with float64 numpy.

The end-to-end tests cannot see these kernels: a wrong candidate score only makes the rank-safety certificate reject
the query, and the exact fallback then returns the right page. Here the scores themselves are checked:
  * integer inputs |x| <= 15 are exact in bf16 and every dot product (< 2^24) is exact in fp32 in any order, so dot / mip
    and l2 scores must EQUAL the reference; a wrong swizzle, descriptor advance, k-block ring slot or tail mask gives
    errors of order one;
  * real inputs rounded to bf16 bound the accumulation alone;
  * fp32 inputs check the error bound the certificate (knn_rescore_kernel) assumes for bf16 candidates;
  * the fused epilogue's survivors must be exactly the keys of the unfused scores at or above the threshold."""
import numpy as np
import pytest

import knn_harness as kh
from nrtsearch_b200 import index as ix

pytestmark = pytest.mark.gpu

SIMS = (ix.SIM_L2, ix.SIM_DOT, ix.SIM_COSINE, ix.SIM_MIP)
# rsqrtf is within 2 ulp, the product with the dot rounds once more: cosine scores of exact dots are within this
# relative error of the float64 quotient
COS_REL = 2.5 * 2.0**-23
# knn_score_upper_bound: candidate-stage error of a bf16 dot product <= eps_rel * (1 + 1e-3) * |q| * dmax
CERT_EPS = 2.0**-7 * (1 + 1e-3)


@pytest.fixture(scope="module")
def harness(built):
    return kh.lib()


def _ints(rng, shape):
    return rng.integers(-15, 16, size=shape).astype(np.float32)


def _assert_integer_exact(S, Q, Dc, sim, what):
    dot = Q.astype(np.float64) @ Dc.astype(np.float64).T          # integers < 2^53: exact
    n2 = (Dc.astype(np.float64) ** 2).sum(axis=1)
    if sim == ix.SIM_COSINE:
        want = dot / np.sqrt(np.maximum(n2, 1e-30))[None, :]
        err = np.abs(S - want)
        assert (err <= COS_REL * np.abs(want)).all(), f"{what}: cosine max rel err {np.max(err / np.maximum(np.abs(want), 1e-30)):.3g}"
        return
    want = 2.0 * dot - n2[None, :] if sim == ix.SIM_L2 else dot
    bad = np.argwhere(S != want)
    assert len(bad) == 0, f"{what}: {len(bad)} scores differ, first at {tuple(bad[0])}: {S[tuple(bad[0])]} vs {want[tuple(bad[0])]}"


def _gemm_integer_case(M, N, K, n_base, n_total, seed):
    rng = np.random.default_rng(seed)
    Q, D = _ints(rng, (M, K)), _ints(rng, (n_total, K))
    Dc = D[n_base:n_base + N]
    for sim in SIMS:
        S = kh.gemm_scores(Q, D, sim, n_base=n_base, N=N)
        _assert_integer_exact(S, Q, Dc, sim, f"gemm M={M} N={N} K={K} n_base={n_base} sim={sim}")


# K: below one 64-column box, one box, partial second box, exactly kStages = 3 k-blocks, a ring that wraps, dims = 4096
@pytest.mark.parametrize("K", [8, 16, 56, 64, 72, 192, 200, 256, 768, 1000, 4096])
def test_gemm_integer_exact_over_k(harness, K):
    _gemm_integer_case(M=130, N=300, K=K, n_base=0, n_total=350, seed=K)


# M around the 64-row warpgroup half and the 128-row tile
@pytest.mark.parametrize("M", [1, 63, 64, 65, 127, 128, 129, 300])
def test_gemm_integer_exact_over_m(harness, M):
    _gemm_integer_case(M=M, N=129, K=72, n_base=0, n_total=200, seed=100 + M)


# N around the 128-column tile, inside a larger corpus (the tile reads real rows past N that must be masked) and at the
# corpus end (the tile runs past the tensor, TMA fills zeros)
@pytest.mark.parametrize("at_end", [False, True])
@pytest.mark.parametrize("N", [1, 127, 128, 129, 1000])
def test_gemm_integer_exact_over_n(harness, N, at_end):
    n_base = 333 if at_end else 0
    _gemm_integer_case(M=65, N=N, K=200, n_base=n_base, n_total=n_base + N if at_end else N + 77, seed=200 + N)


def test_device_bf16_conversion_matches_reference(harness):
    rng = np.random.default_rng(1)
    hi = rng.integers(0, 0x7F7F, 4096).astype(np.uint32) << 16
    x = np.concatenate([rng.standard_normal(100_000).astype(np.float32),
                        (np.concatenate([hi | 0x8000, hi | 0x7FFF, hi | 0x8001])).view(np.float32),
                        kh.below_midpoint(rng, 4096)])
    assert np.array_equal(kh.device_bf16(x).view(np.uint32), kh.bf16_round(x).view(np.uint32))


@pytest.mark.parametrize("kind", ["gauss", "positive"])
@pytest.mark.parametrize("K", [64, 768, 4096])
def test_gemm_accumulation_bound_on_bf16_inputs(harness, K, kind):
    """Against the float64 product of the bf16-ROUNDED inputs the only error left is the fp32 accumulation:
    |S - ref| <= K * 2^-23 * sum |q~_i d~_i| (every product is exact in fp32; K roundings of at most one ulp each)."""
    rng = np.random.default_rng(K)
    if kind == "gauss":
        Q, D = rng.standard_normal((129, K)).astype(np.float32), rng.standard_normal((300, K)).astype(np.float32)
    else:
        Q, D = rng.uniform(0, 1, (129, K)).astype(np.float32), rng.uniform(0, 1, (300, K)).astype(np.float32)
    Qr, Dr = kh.bf16_round(Q).astype(np.float64), kh.bf16_round(D).astype(np.float64)
    S = kh.gemm_scores(Q, D, ix.SIM_DOT)
    ref = Qr @ Dr.T
    absdot = np.abs(Qr) @ np.abs(Dr).T
    err = np.abs(S - ref)
    assert (err <= K * 2.0**-23 * absdot).all(), np.max(err / absdot)


def _certificate_data(kind, dims, rng, M=64, N=1024):
    if kind == "gauss":
        return rng.standard_normal((M, dims)).astype(np.float32), rng.standard_normal((N, dims)).astype(np.float32)
    if kind == "positive":
        return rng.uniform(0, 1, (M, dims)).astype(np.float32), rng.uniform(0, 1, (N, dims)).astype(np.float32)
    if kind == "neardup":   # queries within 1e-3 of corpus rows: sum |q_i d_i| = |q||d| to 1e-6
        D = rng.uniform(0.5, 1.5, (N, dims)).astype(np.float32)
        return (D[:M] * (1 + 1e-3 * rng.standard_normal((M, dims)))).astype(np.float32), D
    # "midpoint": every component just below a bf16 rounding midpoint, queries = corpus rows: every product loses
    # almost 2^-7 of itself to the operand rounding, all in the same direction
    D = kh.below_midpoint(rng, (N, dims))
    return D[:M].copy(), D


@pytest.mark.parametrize("kind", ["gauss", "positive", "neardup", "midpoint"])
@pytest.mark.parametrize("dims", [64, 768, 4096])
def test_gemm_error_within_certificate_bound(harness, dims, kind):
    """The premise of the rank-safety certificate, on fp32 inputs: the bf16 candidate score of every vector is within
    2^-7 (1 + 1e-3) |q| dmax of its exact value (dot / mip), twice that for l2 (2 dot - |d|^2), 2^-7 (1 + 1e-3) |q| for
    cosine (dot / |d|). Prints the measured margin."""
    rng = np.random.default_rng(dims + len(kind))
    Q, D = _certificate_data(kind, dims, rng)
    Q64, D64 = Q.astype(np.float64), D.astype(np.float64)
    qn, dn = np.linalg.norm(Q64, axis=1), np.linalg.norm(D64, axis=1)
    dmax = dn.max()
    worst = {}
    for sim, bound in ((ix.SIM_DOT, CERT_EPS * qn[:, None] * dmax), (ix.SIM_L2, 2 * CERT_EPS * qn[:, None] * dmax),
                       (ix.SIM_COSINE, CERT_EPS * qn[:, None] * np.ones((1, len(D))))):
        err = np.abs(kh.gemm_scores(Q, D, sim) - kh.approx_reference(Q64, D64, sim))
        worst[sim] = float(np.max(err / bound))
        if sim == ix.SIM_DOT:
            rel = float(np.max(err / (qn[:, None] * dn[None, :])))
    print(f"\n[certificate] dims={dims} {kind}: max err/(|q||d|) = {rel:.4e} (2^-7 = {2.0**-7:.4e}); "
          f"err/bound dot {worst[ix.SIM_DOT]:.4f} l2 {worst[ix.SIM_L2]:.4f} cosine {worst[ix.SIM_COSINE]:.4f}")
    assert max(worst.values()) <= 1.0, worst


# ---- fused epilogue: survivors of one chunk ----

def _fused_expected(S, theta, n_base, filter_docs, live_docs, vec_docs):
    M, N = S.shape
    ords = n_base + np.arange(N)
    docs = ords if vec_docs is None else vec_docs[ords]
    ok = np.ones(N, bool)
    if filter_docs is not None:
        ok &= filter_docs[docs] != 0
    if live_docs is not None:
        ok &= live_docs[docs] != 0
    mask = (S >= theta[:, None]) & ok[None, :]
    x = S + np.float32(0.0)   # the epilogue computes a * acc + b with b = +0 for dot / cosine: a zero score is +0
    return [kh.make_key(x[q, mask[q]], ords[mask[q]]) for q in range(M)]


FUSED_CASES = {
    # name: (M, N, n_base, n_total, K, sim, theta, cc_cap, with filter / live / vec_docs)
    "all_survive_spill": (200, 1000, 0, 1000, 64, ix.SIM_COSINE, "none", 1000, False),
    "cc_cap_overflow": (200, 1000, 0, 1000, 64, ix.SIM_DOT, "none", 100, False),
    "theta_filter_live_vecdocs": (129, 1000, 700, 1700, 200, ix.SIM_L2, 40, 1000, True),
    "few_survivors_filtered": (300, 513, 64, 700, 128, ix.SIM_MIP, 5, 600, True),
}


@pytest.mark.parametrize("case", list(FUSED_CASES))
def test_gemm_fused_epilogue_survivors(harness, case):
    """theta = -inf sends far more than kRowCap = 8 survivors per row and tile through the global atomic; a small
    cc_cap makes the chunk count exceed the buffer (the count must stay exact, the stored keys a subset); a theta taken
    from the unfused scores (the k-th best, so ties at theta are included) with filter, deletes and a non-identity
    vec_docs map checks which keys survive."""
    M, N, n_base, n_total, K, sim, th, cc_cap, masks = FUSED_CASES[case]
    rng = np.random.default_rng(len(case) * 7 + M)
    Q = rng.standard_normal((M, K)).astype(np.float32)
    D = rng.standard_normal((n_total, K)).astype(np.float32)
    flt = live = vd = None
    n_docs = n_total
    if masks:
        n_docs = 2 * n_total
        vd = rng.permutation(n_docs)[:n_total].astype(np.int32)
        flt = (rng.random(n_docs) < 0.7).astype(np.uint8)
        live = (rng.random(n_docs) < 0.8).astype(np.uint8)
    S = kh.gemm_scores(Q, D, sim, n_base=n_base, N=N)
    theta = np.full(M, -np.inf, np.float32) if th == "none" else -np.sort(-S, axis=1)[:, th - 1].copy()
    cc, cnt = kh.gemm_fused(Q, D, sim, theta, cc_cap, n_base=n_base, N=N, filter_docs=flt, live_docs=live,
                            vec_docs=vd, n_docs=n_docs)
    want = _fused_expected(S, theta, n_base, flt, live, vd)
    overflowed = 0
    for q in range(M):
        assert cnt[q] == len(want[q]), (q, int(cnt[q]), len(want[q]))
        stored = cc[q, :min(int(cnt[q]), cc_cap)]
        if cnt[q] <= cc_cap:
            assert np.array_equal(np.sort(stored), np.sort(want[q])), q
        else:
            overflowed += 1
            assert len(np.unique(stored)) == cc_cap and np.isin(stored, want[q]).all(), q
    if case == "cc_cap_overflow":
        assert overflowed == M
    if case == "all_survive_spill":
        assert (cnt == N).all()


# ---- fp32 SIMT candidate stage ----

@pytest.mark.parametrize("K", [3, 64, 100, 1001])
def test_dot_tile_integer_exact_and_bound(harness, K):
    """knn_dot_tile_kernel (any dims; the tensor-core stage needs dims % 8 == 0): integer inputs exact for every
    similarity, real inputs within the fp32 FMA chain's bound K * 2^-23 * sum |q_i d_i| of the float64 dot."""
    rng = np.random.default_rng(K)
    M, N = 70, 130                                       # edges of the 64 x 64 tile on both axes
    Q, D = _ints(rng, (M, K)), _ints(rng, (N, K))
    for sim in SIMS:
        _assert_integer_exact(kh.dot_tile_scores(Q, D, sim), Q, D, sim, f"dot_tile K={K} sim={sim}")
    Q, D = rng.standard_normal((M, K)).astype(np.float32), rng.standard_normal((N, K)).astype(np.float32)
    Q64, D64 = Q.astype(np.float64), D.astype(np.float64)
    err = np.abs(kh.dot_tile_scores(Q, D, ix.SIM_DOT) - Q64 @ D64.T)
    assert (err <= K * 2.0**-23 * (np.abs(Q64) @ np.abs(D64).T)).all()
