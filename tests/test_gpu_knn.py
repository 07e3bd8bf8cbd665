"""kNN parity: CUDA exact path vs the oracle's brute force (ExactVectorQuery semantics,
reference VectorFieldDefTest.java:1886-2117 compares exact search with brute force at 1e-4)."""
import numpy as np
import pytest

import knn_harness as kh
import oracle
from nrtsearch_b200 import _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200.index import HostShard, TextField
from nrtsearch_b200.search import GpuIndex, GpuIndexSearcher

pytestmark = pytest.mark.gpu


def vec_shard(vectors, sim, vec_docs=None, n_docs=None, live_docs=None, doc_base=0):
    n = len(vectors) if n_docs is None else n_docs
    return HostShard(n_docs=n, doc_base=doc_base, term_off=np.zeros(1, np.int64), post_docs=np.zeros(0, np.int32),
                     post_freqs=np.zeros(0, np.int32), fields=[], vectors=vectors, vec_similarity=sim, vec_docs=vec_docs,
                     live_docs=live_docs)


def check(gd, gs, gc, wd, ws, wc, rtol=1e-5):
    """Parity spec for the vector path (SURVEY.md 8c): identical counts; scores within 1e-5 relative (the GPU re-score
    and the oracle both accumulate in fp64, but in different orders); doc ids identical EXCEPT inside a tie band:
    positions i whose oracle scores lie within rtol of each other may be permuted, nothing else. The tie band is
    explicit: every differing position must hold a doc that the oracle ranks at a position whose score is within rtol."""
    assert np.array_equal(gc, wc)
    for q in range(len(gc)):
        n = int(gc[q])
        np.testing.assert_allclose(gs[q, :n], ws[q, :n], rtol=rtol, atol=0)
        if np.array_equal(gd[q, :n], wd[q, :n]):
            continue
        pos = {int(d): i for i, d in enumerate(wd[q, :n])}
        for i in np.nonzero(gd[q, :n] != wd[q, :n])[0]:
            d = int(gd[q, i])
            if d in pos:   # permuted inside the list: the two positions must be a score tie within tolerance
                assert abs(ws[q, pos[d]] - ws[q, i]) <= rtol * abs(ws[q, i]), (q, i, d)
            else:          # swapped with a doc just outside the oracle's list: only legal at the boundary tie
                assert abs(gs[q, i] - ws[q, n - 1]) <= rtol * abs(ws[q, n - 1]), (q, i, d)


def kprime(k, tensor_core=True):
    """Candidates kept per query by knn_search_host: 4k (at least 128) for the bf16 stage, 2k (at least 64) for fp32."""
    kp = max(128, 4 * k) if tensor_core else max(64, 2 * k)
    return min(kp, 4096 - 256)


def assert_certifiable(corpus, queries, sim, k, tensor_core=True, eligible=None):
    """The exact gap between every query's k-th and k'-th best candidate scores (among eligible vectors) clearly
    exceeds the candidate stage's error bound, so a correct candidate stage must certify every query: the bf16 bound
    2^-7 (1 + 1e-3) |q| dmax (twice that for l2, |q| for cosine), or dims * 2^-23 for the fp32 stage."""
    corpus = np.asarray(corpus, np.float64)
    kp = kprime(k, tensor_core)
    n_ok = len(corpus) if eligible is None else int(np.count_nonzero(eligible))
    assert n_ok > kp, "the candidate list must be full for the certificate to matter"
    eps = (2.0**-7 if tensor_core else corpus.shape[1] * 2.0**-23) * (1 + 1e-3)
    dmax = np.linalg.norm(corpus, axis=1).max()
    for q0 in range(0, len(queries), 16):
        qs = np.asarray(queries[q0:q0 + 16], np.float64)
        a = kh.approx_reference(qs, corpus, sim)
        if eligible is not None:
            a[:, ~np.asarray(eligible, bool)] = -np.inf
        top = -np.partition(-a, [k - 1, kp - 1], axis=1)
        gap = top[:, k - 1] - top[:, kp - 1]
        qn = np.linalg.norm(qs, axis=1)
        bound = eps * qn * ({ix.SIM_L2: 2 * dmax, ix.SIM_COSINE: 1.0}.get(sim, dmax))
        assert (gap > 3 * bound).all(), np.min(gap / bound)


@pytest.mark.parametrize("sim", [ix.SIM_L2, ix.SIM_COSINE, ix.SIM_MIP])
def test_knn_matches_bruteforce(gpu_ctx, sim):
    corpus = ix.synth_vectors(20_000, 96)
    queries = ix.synth_vectors(50, 96, seed=ix.SEED_VQUERIES)
    gix = GpuIndex(gpu_ctx, vec_shard(corpus, sim))
    gd, gs, gc = GpuIndexSearcher(gix).knn(queries, 10)
    gix.close()
    wd, ws, wc = oracle.knn_exact(corpus, sim, queries, 10)
    check(gd, gs, gc, wd, ws, wc)


def test_knn_normalized_dot_product_filter_boost(gpu_ctx):
    corpus = ix.synth_vectors(5_000, 64)
    corpus /= np.linalg.norm(corpus, axis=1, keepdims=True)
    queries = ix.synth_vectors(20, 64, seed=ix.SEED_VQUERIES)
    queries /= np.linalg.norm(queries, axis=1, keepdims=True)
    flt = (np.arange(5000) % 3 == 0).astype(np.uint8)
    boosts = np.linspace(0.5, 2.0, 20).astype(np.float32)
    gix = GpuIndex(gpu_ctx, vec_shard(corpus.astype(np.float32), ix.SIM_DOT))
    gd, gs, gc = GpuIndexSearcher(gix).knn(queries, 25, boosts=boosts, filter_docs=flt)
    gix.close()
    wd, ws, wc = oracle.knn_exact(corpus, ix.SIM_DOT, queries, 25, filter_docs=flt, boosts=boosts)
    check(gd, gs, gc, wd, ws, wc)
    assert (gd % 3 == 0).all()


def test_knn_fewer_vectors_than_k(gpu_ctx):
    corpus = ix.synth_vectors(7, 16)
    queries = ix.synth_vectors(3, 16, seed=ix.SEED_VQUERIES)
    gix = GpuIndex(gpu_ctx, vec_shard(corpus, ix.SIM_COSINE))
    gd, gs, gc = GpuIndexSearcher(gix).knn(queries, 10)
    gix.close()
    wd, ws, wc = oracle.knn_exact(corpus, ix.SIM_COSINE, queries, 10)
    assert list(gc) == [7, 7, 7]
    check(gd, gs, gc, wd, ws, wc)


def test_knn_768_dims_tensor_core_path(gpu_ctx):
    # C4 shape at reduced N: 768-d cosine, top-100; the bf16 tensor-core stage only picks candidates, the exact
    # re-score must reproduce the oracle's ids and scores (recall 1.0 expected)
    corpus = ix.synth_vectors(30_000, 768)
    queries = ix.synth_vectors(130, 768, seed=ix.SEED_VQUERIES)   # not a multiple of the 128-row MMA tile
    gix = GpuIndex(gpu_ctx, vec_shard(corpus, ix.SIM_COSINE))
    gd, gs, gc = GpuIndexSearcher(gix).knn(queries, 100)
    gix.close()
    wd, ws, wc = oracle.knn_exact(corpus, ix.SIM_COSINE, queries, 100)
    recall = np.mean([len(set(gd[q]) & set(wd[q])) / 100.0 for q in range(len(queries))])
    assert recall >= 0.999, recall
    check(gd, gs, gc, wd, ws, wc)


def test_knn_excludes_deleted_docs(gpu_ctx):
    # ExactVectorQuery / KnnFloatVectorQuery never return deleted docs (IndexSearcher acceptDocs); filter ANDs on top
    corpus = ix.synth_vectors(12_000, 64)
    queries = ix.synth_vectors(40, 64, seed=ix.SEED_VQUERIES)
    live = np.ones(12_000, np.uint8)
    live[::3] = 0
    flt = (np.arange(12_000) % 5 != 0).astype(np.uint8)
    gix = GpuIndex(gpu_ctx, vec_shard(corpus, ix.SIM_COSINE, live_docs=live))
    s = GpuIndexSearcher(gix)
    gd, gs, gc = s.knn(queries, 20)
    gd2, gs2, gc2 = s.knn(queries, 20, filter_docs=flt)
    gix.close()
    wd, ws, wc = oracle.knn_exact(corpus, ix.SIM_COSINE, queries, 20, live_docs=live)
    check(gd, gs, gc, wd, ws, wc)
    assert (gd % 3 != 0).all()
    wd2, ws2, wc2 = oracle.knn_exact(corpus, ix.SIM_COSINE, queries, 20, live_docs=live, filter_docs=flt)
    check(gd2, gs2, gc2, wd2, ws2, wc2)
    assert (gd2 % 3 != 0).all() and (gd2 % 5 != 0).all()


def test_knn_rank_safe_on_near_duplicates(gpu_ctx):
    """Adversarial for a bf16 candidate stage: thousands of vectors within 1e-4 of the query direction (score gaps far
    below the bf16 error 2^-7). The certificate must reject the candidate list and the exact fallback must return
    the oracle's ids (ExactVectorQuery semantics: exact by construction, not by luck)."""
    from nrtsearch_b200 import _native
    rng = np.random.default_rng(7)
    dims, n = 128, 40_000
    base = rng.standard_normal(dims).astype(np.float32)
    corpus = ix.synth_vectors(n, dims)
    near = rng.choice(n, size=3000, replace=False)
    corpus[near] = base[None, :] * (1.0 + rng.uniform(0, 0.5, size=(3000, 1))).astype(np.float32) \
        + 1e-4 * rng.standard_normal((3000, dims)).astype(np.float32)
    queries = np.stack([base + 1e-4 * rng.standard_normal(dims).astype(np.float32) for _ in range(6)]
                       + [ix.synth_vectors(1, dims, seed=99)[0] for _ in range(2)]).astype(np.float32)
    for sim in (ix.SIM_COSINE, ix.SIM_L2, ix.SIM_MIP):
        gix = GpuIndex(gpu_ctx, vec_shard(corpus, sim))
        gd, gs, gc = GpuIndexSearcher(gix).knn(queries, 50)
        unc = _native.gpu_lib().nrtgpu_knn_last_uncertified(gix.handle)
        gix.close()
        wd, ws, wc = oracle.knn_exact(corpus, sim, queries, 50)
        check(gd, gs, gc, wd, ws, wc)
        if sim == ix.SIM_COSINE:
            assert unc >= 6, unc   # the six near-duplicate queries cannot be certified from bf16 scores


@pytest.mark.parametrize("sim", [ix.SIM_L2, ix.SIM_DOT, ix.SIM_COSINE, ix.SIM_MIP])
def test_knn_byte_vectors(gpu_ctx, sim):
    """ByteVectorFieldDef (VectorFieldDef.java:870-881): int8 vectors, byte score mapping (DOT_PRODUCT = 0.5 + dot / (dims * 2^15))."""
    rng = np.random.default_rng(11 + sim)
    corpus = rng.integers(-128, 128, size=(9_000, 96), dtype=np.int8)
    queries = rng.integers(-128, 128, size=(30, 96), dtype=np.int8).astype(np.float32)
    gix = GpuIndex(gpu_ctx, vec_shard(corpus, sim))
    gd, gs, gc = GpuIndexSearcher(gix).knn(queries, 20)
    gix.close()
    wd, ws, wc = oracle.knn_exact(corpus.astype(np.float32), sim | 0x100, queries, 20)
    check(gd, gs, gc, wd, ws, wc)


def test_knn_normalized_cosine(gpu_ctx):
    """nrtsearch's normalized_cosine (VectorFieldDef.java:308-332, 568-573, 651-655): vectors are L2-normalised at index and
    query time (float division by the float magnitude), searched with DOT_PRODUCT; the magnitude goes to <field>._magnitude."""
    from nrtsearch_b200.search import normalized_cosine_vectors
    raw = ix.synth_vectors(8_000, 80) * 3.0
    queries = ix.synth_vectors(25, 80, seed=ix.SEED_VQUERIES) * 0.2
    unit, magnitude = normalized_cosine_vectors(raw)
    qunit, _ = normalized_cosine_vectors(queries)
    assert np.allclose(np.linalg.norm(unit, axis=1), 1.0, atol=1e-5) and np.allclose(magnitude, np.linalg.norm(raw, axis=1), rtol=1e-5)
    gix = GpuIndex(gpu_ctx, vec_shard(unit, ix.SIM_DOT))
    gd, gs, gc = GpuIndexSearcher(gix).knn(qunit, 30)
    gix.close()
    wd, ws, wc = oracle.knn_exact(unit, ix.SIM_DOT, qunit, 30)
    check(gd, gs, gc, wd, ws, wc)
    cd, cs, cc = oracle.knn_exact(raw, ix.SIM_COSINE, queries, 30)   # and it IS cosine similarity of the raw vectors
    np.testing.assert_allclose(gs, cs, rtol=2e-5)


def knn_run(ctx, shard, queries, k, **kw):
    """GpuIndexSearcher.knn on a fresh index image; also returns how many queries took the exact fallback."""
    gix = GpuIndex(ctx, shard)
    try:
        gd, gs, gc = GpuIndexSearcher(gix).knn(queries, k, **kw)
        unc = _native.gpu_lib().nrtgpu_knn_last_uncertified(gix.handle)
    finally:
        gix.close()
    return gd, gs, gc, unc


def test_knn_fused_chunk_schedule(gpu_ctx):
    """500K vectors: the 32K unfused warm chunk, then fused chunks of 64K, 128K, 256K and a partial second 256K chunk
    ending inside a 128-vector tile; filter, deletes and boosts; 300 queries = three 128-row query tiles. Certified:
    the fused candidate stage alone must find the oracle's page."""
    n, dims, k, nq = 500_000, 16, 10, 300
    corpus = ix.synth_vectors(n, dims)
    queries = ix.synth_vectors(nq, dims, seed=ix.SEED_VQUERIES)
    rng = np.random.default_rng(21)
    live = (rng.random(n) < 0.9).astype(np.uint8)
    flt = (rng.random(n) < 0.8).astype(np.uint8)
    boosts = rng.uniform(0.5, 2.0, nq).astype(np.float32)
    assert_certifiable(corpus, queries, ix.SIM_MIP, k, eligible=(live & flt) != 0)
    gd, gs, gc, unc = knn_run(gpu_ctx, vec_shard(corpus, ix.SIM_MIP, live_docs=live), queries, k, boosts=boosts,
                              filter_docs=flt)
    wd, ws, wc = oracle.knn_exact(corpus, ix.SIM_MIP, queries, k, filter_docs=flt, boosts=boosts, live_docs=live)
    check(gd, gs, gc, wd, ws, wc)
    assert unc == 0, unc


@pytest.mark.parametrize("k", [256, 257, 1024])
def test_knn_unfused_multi_chunk(gpu_ctx, k):
    """k' = 4k > 1024 turns the fused epilogue off (k = 257: k' = 1028; k = 1024 = kMaxTopK: k' capped at 3840); k = 256
    is the last fused k. 150K vectors = three 64K chunks of stored scores, the last one partial."""
    n, dims, nq = 150_000, 32, 130
    corpus = ix.synth_vectors(n, dims)
    queries = ix.synth_vectors(nq, dims, seed=ix.SEED_VQUERIES)
    assert_certifiable(corpus, queries, ix.SIM_COSINE, k)
    gd, gs, gc, unc = knn_run(gpu_ctx, vec_shard(corpus, ix.SIM_COSINE), queries, k)
    wd, ws, wc = oracle.knn_exact(corpus, ix.SIM_COSINE, queries, k)
    check(gd, gs, gc, wd, ws, wc)
    assert unc == 0, unc


@pytest.mark.parametrize("dims, sim, force", [(3, ix.SIM_COSINE, False), (100, ix.SIM_L2, False), (96, ix.SIM_MIP, True)])
def test_knn_simt_candidate_stage(gpu_ctx, monkeypatch, dims, sim, force):
    """knn_dot_tile_kernel: dims % 8 != 0 (no TMA row pitch) or NRTGPU_KNN_SIMT=1; two 32K chunks."""
    if force:
        monkeypatch.setenv("NRTGPU_KNN_SIMT", "1")
    n, k, nq = 40_000, 10, 70
    corpus = ix.synth_vectors(n, dims)
    queries = ix.synth_vectors(nq, dims, seed=ix.SEED_VQUERIES)
    assert_certifiable(corpus, queries, sim, k, tensor_core=False)
    gd, gs, gc, unc = knn_run(gpu_ctx, vec_shard(corpus, sim), queries, k)
    wd, ws, wc = oracle.knn_exact(corpus, sim, queries, k)
    check(gd, gs, gc, wd, ws, wc)
    assert unc == 0, unc


def test_knn_fused_overflow_reruns_without_fusion(gpu_ctx):
    """A filter rejecting every vector of the 32K warm chunk leaves every threshold at -inf, so all 65 536 vectors of
    the first fused chunk survive and overflow the 3072-key chunk buffer: the search reruns on the fp32 stage."""
    n, dims, k = 100_000, 64, 10
    corpus = ix.synth_vectors(n, dims)
    queries = ix.synth_vectors(20, dims, seed=ix.SEED_VQUERIES)
    flt = (np.arange(n) >= 32768).astype(np.uint8)
    gd, gs, gc, _ = knn_run(gpu_ctx, vec_shard(corpus, ix.SIM_L2), queries, k, filter_docs=flt)
    wd, ws, wc = oracle.knn_exact(corpus, ix.SIM_L2, queries, k, filter_docs=flt)
    check(gd, gs, gc, wd, ws, wc)
    assert (gd >= 32768).all()


def test_knn_sparse_vec_docs_and_doc_base(gpu_ctx):
    """A sparse vector field (vec_docs: ascending ordinal -> doc over twice as many docs) in a leaf with doc_base != 0;
    filter and deletes are per doc. The oracle searches ordinals: filter and live map to ordinals, its ordinals to docs."""
    n_vec, dims, k, nq, doc_base = 70_000, 32, 20, 40, 1_000_000
    n_docs = 2 * n_vec
    rng = np.random.default_rng(33)
    vec_docs = np.sort(rng.choice(n_docs, n_vec, replace=False)).astype(np.int32)
    corpus = ix.synth_vectors(n_vec, dims)
    queries = ix.synth_vectors(nq, dims, seed=ix.SEED_VQUERIES)
    live = (rng.random(n_docs) < 0.9).astype(np.uint8)
    flt = (rng.random(n_docs) < 0.85).astype(np.uint8)
    assert_certifiable(corpus, queries, ix.SIM_COSINE, k, eligible=(live[vec_docs] & flt[vec_docs]) != 0)
    shard = vec_shard(corpus, ix.SIM_COSINE, vec_docs=vec_docs, n_docs=n_docs, live_docs=live, doc_base=doc_base)
    gd, gs, gc, unc = knn_run(gpu_ctx, shard, queries, k, filter_docs=flt)
    wo, ws, wc = oracle.knn_exact(corpus, ix.SIM_COSINE, queries, k, filter_docs=flt[vec_docs], live_docs=live[vec_docs])
    wd = np.where(np.arange(k)[None, :] < wc[:, None], vec_docs[np.clip(wo, 0, n_vec - 1)] + doc_base, 0)
    check(gd, gs, gc, wd, ws, wc)
    assert unc == 0, unc
