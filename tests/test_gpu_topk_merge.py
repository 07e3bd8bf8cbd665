"""The relevance top-k kernels against tests/topk_reference.py, exactly (docs equal, scores bit for bit, counts, totals and
flags equal), at the shapes where they go wrong:

- merge_slices_kernel (the per-query merge of a batch's work-item lists, through tests/csrc/topk_harness.cu): 1 to 600
  lists across its 256-list chunks of counts, top_k 1 to 1024, empty / sparse / full lists and runs that end exactly at its
  4096-key buffer, thresholds, doc_base, and every flag and total input;
- flush_top_k (the posting kernels' candidate cut and threshold publication) at the probe kernel's and the window engine's
  buffer sizes;
- merge_pairs_kernel (TopDocs.merge over leaves and GPUs) through nrtgpu_merge_topk_packed and nrtgpu_merge_topk_device;
- rrf_blend_kernel and rescore_combine_kernel at their 4096-key limit, and the refusals past it.

Every page of k slots holds its hits first and doc 0 / score 0.0 past its count, whatever the buffer held before: the
device outputs start as a sentinel, and the host outputs of the pooled buffers are checked after a call with more hits."""
import ctypes
import itertools

import numpy as np
import pytest

import oracle
import topk_harness as th
import topk_reference as ref
from nrtsearch_b200 import _native
from nrtsearch_b200.search import blend_rrf, blend_scores, rescore_combine

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
# scores with ties, both signs, subnormals and +inf (no -0.0: its order against +0.0 is not Lucene's)
SCORES = np.concatenate([np.float32([np.inf, 3.4028235e38, 1e-40, 1e-45, 0.0, -1e-45, -1e-40, -3.4028235e38]),
                         np.linspace(-8, 8, 24).astype(np.float32)])
# retriever and first-pass scores: a boost or weight times a negative score could make -0.0
BLEND_SCORES = SCORES[(SCORES >= 0) & (SCORES < 1e30)]
PATTERNS = ("empty", "sparse", "full", "flat4096")


def _assert_pages(docs, scores, counts, want, what):
    """docs / scores [nq, k] and counts [nq] against want: one (docs, scores) page per query, padded with doc 0 / 0.0"""
    k = docs.shape[1]
    for q, (wd, ws) in enumerate(want):
        ed, es = ref.padded(wd, ws, k)
        assert counts[q] == len(wd), (what, q, counts[q], len(wd))
        assert np.array_equal(docs[q], ed), (what, q, np.flatnonzero(docs[q] != ed)[:5])
        assert np.array_equal(scores[q].view(np.uint32), es.view(np.uint32)), (what, q)


def _counts(rng, pattern, n_lists, top_k):
    c = np.zeros(n_lists, np.int32)
    if pattern == "sparse":   # most work items of a query end empty; non-empty lists on both sides of 255 / 256
        pick = rng.choice(n_lists, max(1, n_lists // 16), replace=False)
        pick = np.concatenate([pick, [l for l in (0, 254, 255, 256, 257, n_lists - 1) if l < n_lists]])
        c[pick] = rng.integers(1, top_k + 1, len(pick))
    elif pattern == "full":
        c[:] = top_k
    elif pattern == "flat4096":   # lists that fill the merge buffer exactly, then one key more
        need = -(-4096 // top_k)
        l = max(0, min(250, n_lists - need - 1))
        left = 4096
        while left > 0 and l < n_lists:
            c[l] = min(top_k, left)
            left -= c[l]
            l += 1
        if l < n_lists:
            c[l] = 1
    return c


def _slice_lists(rng, nq, n_lists, top_k, doc_base):
    """per query: lists [n_lists, top_k] of distinct docs (>= 1, some near INT32_MAX - doc_base), ordered best first as
    a flush leaves them; the keys past a list's count are junk the merge must not read"""
    counts = np.stack([_counts(rng, PATTERNS[q % 4], n_lists, top_k) for q in range(nq)])
    n = n_lists * top_k
    docs = np.empty((nq, n_lists, top_k), np.int32)
    for q in range(nq):
        d = 1 + rng.permutation(2 * n)[:n]
        docs[q] = (d if q % 2 else INT_MAX - doc_base - d).reshape(n_lists, top_k)
    scores = rng.choice(SCORES, (nq, n_lists, top_k))
    keys = ref.make_keys(scores, docs)
    o = np.argsort(keys, axis=2)[:, :, ::-1]
    keys, docs, scores = (np.take_along_axis(a, o, axis=2) for a in (keys, docs, scores))
    keys[np.arange(top_k)[None, None, :] >= counts[:, :, None]] = np.uint64(2**64 - 1)
    return keys, docs, scores, counts


def _theta(mode, docs, scores, counts, top_k):
    """a query's threshold pair: None (mode 0), the k-th best pair present (mode 1: kept, >=), or a pair above all (mode 2)"""
    m = np.arange(top_k)[None, :] < counts[:, None]
    s, d = scores[m], docs[m]
    if mode == 0 or len(s) == 0:
        return None
    o = ref.order(s, d)
    if mode == 1:
        i = o[min(top_k, len(o)) - 1]
        return float(s[i]), int(d[i])
    return float(s[o[0]]), int(d[o[0]]) - 1   # docs are >= 1


def _flag_inputs(nq):
    """every combination of counted total (around terminate_after = 1000), pruned, terminated and known hits"""
    combos = list(itertools.product([0, 999, 1000, 1001, 2**40], [0, 1], [0, 1], [0, 500, 5000, 2**41]))
    c = np.array([combos[q % len(combos)] for q in range(nq)], np.int64)
    return c[:, 0].astype(np.uint64), c[:, 1].astype(np.int32), c[:, 2].astype(np.int32), c[:, 3].astype(np.uint64)


@pytest.mark.parametrize("top_k", [1, 100, 1000, 1024])
@pytest.mark.parametrize("n_lists", [1, 33, 255, 256, 257, 321, 600])
def test_merge_slices(built, n_lists, top_k):
    rng = np.random.default_rng(n_lists * 7919 + top_k)
    n = n_lists * top_k
    nq = 1100 if n <= 3300 else max(12, min(80, 3_000_000 // n))
    doc_base = 0 if top_k == 100 else 1_000_003
    keys, docs, scores, counts = _slice_lists(rng, nq, n_lists, top_k, doc_base)
    # no optional input
    out = th.merge_slices(keys, counts, top_k, doc_base)
    want = [ref.merge_slices_page(scores[q], docs[q], counts[q], top_k, doc_base) for q in range(nq)]
    _assert_pages(out["docs"], out["scores"], out["counts"], want, "bare")
    # thresholds and the whole flag / total matrix
    thetas = [_theta(q % 3, docs[q], scores[q], counts[q], top_k) for q in range(nq)]
    tkeys = np.array([0 if t is None else ref.make_keys([t[0]], [t[1]])[0] for t in thetas], np.uint64)
    total, pruned, term, known = _flag_inputs(nq)
    out = th.merge_slices(keys, counts, top_k, doc_base, theta=tkeys, total_hits=total, pruned=pruned, terminated=term,
                          terminate_after=1000, known_hits=known, want_total=True, want_flags=True)
    want = [ref.merge_slices_page(scores[q], docs[q], counts[q], top_k, doc_base, thetas[q]) for q in range(nq)]
    _assert_pages(out["docs"], out["scores"], out["counts"], want, "theta")
    wterm, wtotal, wflags = ref.merge_slices_flags(total, pruned, term, 1000, known, nq)
    assert np.array_equal(out["terminated"], wterm) and np.array_equal(out["total"], wtotal) and np.array_equal(out["flags"], wflags)
    # totals and flags without the optional inputs
    out = th.merge_slices(keys[:4], counts[:4], top_k, doc_base, want_total=True, want_flags=True)
    assert not out["total"].any() and not out["flags"].any()


def test_merge_slices_refuses_what_no_producer_makes(built):
    keys = ref.make_keys(np.ones((1, 2, 4), np.float32), np.arange(8).reshape(1, 2, 4) + 1)
    zero = keys.copy()
    zero[0, 1, 0] = 0
    wide = ref.make_keys(np.ones((1, 1, 1025), np.float32), np.arange(1025).reshape(1, 1, 1025) + 1)
    for k, c, kk, base in ((keys, [[5, 0]], 4, 0), (keys, [[-1, 0]], 4, 0), (zero, [[4, 1]], 4, 0), (keys, [[4, 1]], 4, INT_MAX),
                           (wide, [[1]], 1025, 0)):
        with pytest.raises(th.HarnessError) as e:
            th.merge_slices(k, c, kk, base)
        assert e.value.rc == th.INVALID


@pytest.mark.parametrize("cap,n_threads,top_k", [(1024, 256, 1), (1024, 256, 100), (1024, 256, 1024), (4096, 512, 1),
                                                 (4096, 512, 100), (4096, 512, 1024)])
def test_flush_top_k(built, cap, n_threads, top_k):
    rng = np.random.default_rng(cap + top_k)
    for count in sorted({0, 1, top_k - 1, top_k, top_k + 1, cap, cap + 37}):
        for dec in (0, 1):
            for prior in ("below", "above"):
                docs = (1 + rng.permutation(4 * cap)[:cap]).astype(np.int32)
                scores = rng.choice(SCORES, cap)
                cand = ref.make_keys(scores, docs)
                cand[min(count, cap):] = np.uint64(2**64 - 1)   # past the count: never read
                wd, ws, _, _, _ = ref.flush(scores, docs, count, cap, top_k, dec, 0, 0)
                kth = int(ref.make_keys(ws[-1:], wd[-1:])[0]) if len(wd) else 1 << 40
                g0 = kth - 1000 if prior == "below" else kth + 1000
                t0 = g0 // 2
                buf, n, g, t = th.flush_top_k(cand, count, cap, top_k, dec, g0, t0, n_threads)
                wd, ws, wn, wg, wt = ref.flush(scores, docs, count, cap, top_k, dec, g0, t0)
                what = (count, dec, prior)
                assert n == wn and g == wg and t == wt, what
                assert np.array_equal(buf[:n], ref.make_keys(ws, wd)), what


def test_flush_top_k_refuses_what_no_producer_makes(built):
    cand = np.zeros(1024, np.uint64)
    for cap, count, top_k, dec in ((1000, 0, 10, 0), (8192, 0, 10, 0), (64, 0, 100, 0), (1024, 1, 10, 0), (1024, 0, 10, 2)):
        with pytest.raises(th.HarnessError) as e:
            th.flush_top_k(np.resize(cand, cap), count, cap, top_k, dec, 0, 0, 256)
        assert e.value.rc == th.INVALID


def _packed_words(nq, k):
    w = 2 * nq * k + 2 * nq
    return ((w + 1) & ~1) + 2 * nq


def _pack(docs, scores, counts, flags, totals, nq, k):
    """one packed score record per list (include/nrtgpu.h): docs | scores | counts | flags | pad | totalHits int64"""
    n = nq * k
    rec = np.zeros((len(docs), _packed_words(nq, k)), np.int32)
    w = (2 * n + 2 * nq + 1) & ~1
    for l in range(len(docs)):
        rec[l, :n] = docs[l].reshape(-1)
        rec[l, n:2 * n] = scores[l].reshape(-1).view(np.int32)
        rec[l, 2 * n:2 * n + nq] = counts[l]
        rec[l, 2 * n + nq:2 * n + 2 * nq] = flags[l]
        rec[l, w:w + 2 * nq] = totals[l].astype(np.int64).view(np.int32)
    return rec


@pytest.mark.parametrize("k", [1, 40, 1023, 1024])
@pytest.mark.parametrize("n_lists", [1, 2, 3, 5, 8, 9, 64])
def test_merge_pairs(gpu_ctx, n_lists, k):
    import torch
    rng = np.random.default_rng(n_lists * 31 + k)
    nq = 1100 if k == 40 else 6
    docs = np.stack([(1 + rng.permutation(n_lists * k * 4)[:n_lists * k]).reshape(n_lists, k) for _ in range(nq)], axis=1)
    scores = rng.choice(SCORES, (n_lists, nq, k))
    o = np.argsort(ref.make_keys(scores, docs), axis=2)[:, :, ::-1]
    docs = np.take_along_axis(docs, o, axis=2).astype(np.int32)
    scores = np.take_along_axis(scores, o, axis=2).astype(np.float32)
    counts = rng.integers(0, k + 1, (n_lists, nq)).astype(np.int32)   # mixed; then all empty, all full
    counts[:, 0::3] = 0
    counts[:, 1::3] = k
    totals = rng.integers(INT_MAX - 1000, INT_MAX + 1, (n_lists, nq)).astype(np.int64)
    flags = rng.integers(0, 8, (n_lists, nq)).astype(np.int32)
    wd, ws, wc, wt, wf = ref.merge_pairs(docs, scores, counts, k, totals, flags)
    want = [(wd[q, :wc[q]], ws[q, :wc[q]]) for q in range(nq)]
    dev = torch.device("cuda", 0)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    lib = _native.gpu_lib()
    # nrtgpu_merge_topk_packed
    assert lib.nrtgpu_packed_words(nq, k) == _packed_words(nq, k)
    d_in = torch.from_numpy(_pack(docs, scores, counts, flags, totals, nq, k).reshape(-1)).to(dev)
    d_out = torch.full((_packed_words(nq, k),), th.SENTINEL, dtype=torch.int32, device=dev)
    _native.check(lib.nrtgpu_merge_topk_packed(gpu_ctx.handle, n_lists, nq, k, d_in.data_ptr(), d_out.data_ptr(), stream))
    torch.cuda.synchronize()
    r = d_out.cpu().numpy()
    n, w = nq * k, (2 * nq * k + 2 * nq + 1) & ~1
    _assert_pages(r[:n].reshape(nq, k), r[n:2 * n].view(np.float32).reshape(nq, k), r[2 * n:2 * n + nq], want, "packed")
    assert np.array_equal(r[2 * n + nq:2 * n + 2 * nq], wf)
    assert np.array_equal(r[w:w + 2 * nq].view(np.int64), wt)
    # nrtgpu_merge_topk_device
    td, ts, tc = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (docs, scores, counts))
    od = torch.full((nq * k,), th.SENTINEL, dtype=torch.int32, device=dev)
    os_ = torch.full((nq * k,), th.SENTINEL, dtype=torch.int32, device=dev)
    oc = torch.full((nq,), th.SENTINEL, dtype=torch.int32, device=dev)
    _native.check(lib.nrtgpu_merge_topk_device(gpu_ctx.handle, n_lists, nq, k, td.data_ptr(), ts.data_ptr(), tc.data_ptr(),
                                               od.data_ptr(), os_.data_ptr(), oc.data_ptr(), stream))
    torch.cuda.synchronize()
    _assert_pages(od.cpu().numpy().reshape(nq, k), os_.cpu().numpy().view(np.float32).reshape(nq, k), oc.cpu().numpy(), want,
                  "device")


def _blend_inputs(rng, R, top_in, tie):
    """[R, nq, top_in] docs and scores, counts [R, nq] for 4 queries: every doc in every retriever (heads = top_in), all
    docs distinct (heads = R * top_in), all counts 0, random counts. tie: retriever 1 lists retriever 0's docs in reverse,
    so with equal boosts (and boost 0 for the others) every RRF sum ties with another doc's and doc asc decides."""
    docs = np.zeros((R, 4, top_in), np.int32)
    for r in range(R):
        docs[r, 0] = 1 + rng.permutation(top_in)
        docs[r, 1] = 1 + r * top_in + rng.permutation(top_in)
        docs[r, 2] = rng.permutation(top_in)
        docs[r, 3] = rng.permutation(2 * top_in)[:top_in]
    if tie and R > 1:
        docs[1, 0] = docs[0, 0][::-1]
    counts = np.full((R, 4), top_in, np.int32)
    counts[:, 2] = 0
    counts[:, 3] = rng.integers(0, top_in + 1, R)
    scores = np.sort(rng.choice(BLEND_SCORES, (R, 4, top_in)), axis=2)[:, :, ::-1].copy()
    return docs, scores, counts


@pytest.mark.parametrize("R,top_in", [(1, 4096), (4, 1024), (64, 64)])
def test_blend_at_capacity(gpu_ctx, R, top_in):
    rng = np.random.default_rng(R * 1000 + top_in)
    for tie in (False, True):
        docs, scores, counts = _blend_inputs(rng, R, top_in, tie)
        boosts = (np.float32([1.0, 1.0] + [0.0] * (R - 2))[:R] if R > 1 else np.float32([0.0])) if tie else \
            rng.choice(np.float32([1.0, 0.5, 2.0, 0.7]), R).astype(np.float32)
        for top_out in sorted({1, top_in, 4096, 4097}):
            runs = [(0, rc) for rc in (0, 1, 10**6)] + [(mode, 0) for mode in (1, 2, 3)]
            for mode, rc in runs:
                if mode == 0:
                    d, s, c, t = blend_rrf(gpu_ctx, docs, counts, boosts, rc, top_out)
                else:
                    d, s, c, t = blend_scores(gpu_ctx, {1: "max", 2: "sum", 3: "avg"}[mode], docs, scores, counts, boosts, top_out)
                want = [ref.blend(mode, docs[:, q], counts[:, q], boosts, top_out, scores=scores[:, q], rank_constant=rc)
                        for q in range(4)]
                what = (tie, top_out, mode, rc)
                assert t.tolist() == [w[2] for w in want], what
                _assert_pages(d, s, c, [(w[0], w[1]) for w in want], what)
                if tie and mode == 0 and top_out > 1:
                    assert (np.diff(s[0, :c[0]]) == 0).any(), "no exact tie"


def test_rescore_combine_at_capacity(gpu_ctx):
    rng = np.random.default_rng(4096)
    nq, n = 3, 4096
    docs = np.stack([rng.permutation(3 * n)[:n] for _ in range(nq)]).astype(np.int32)
    scores = np.sort(rng.choice(BLEND_SCORES, (nq, n)), axis=1)[:, ::-1].copy()
    m = (rng.random((nq, n)) < 0.5).astype(np.uint8)
    s2 = rng.choice(np.linspace(0, 2, 30).astype(np.float32), (nq, n))
    for counts in (None, np.array([n, 0, 1234], np.int32)):
        d, s = rescore_combine(gpu_ctx, docs, scores, m, s2, 0.3, 1.7, counts=counts)
        for q in range(nq):
            wd, ws = ref.rescore_combine(docs[q], scores[q], m[q], s2[q], 0.3, 1.7, None if counts is None else counts[q])
            assert np.array_equal(d[q], wd) and np.array_equal(s[q].view(np.uint32), ws.view(np.uint32)), (counts is None, q)


def test_hybrid_refuses_more_than_4096_keys(gpu_ctx):
    for R, top_in in ((1, 4097), (17, 241)):
        docs = np.zeros((R, 1, top_in), np.int32)
        with pytest.raises(_native.NrtGpuUnsupported):
            blend_rrf(gpu_ctx, docs, np.zeros((R, 1), np.int32), [1.0] * R, 60, 10)
        with pytest.raises(_native.NrtGpuUnsupported):
            blend_scores(gpu_ctx, "sum", docs, np.zeros((R, 1, top_in), np.float32), np.zeros((R, 1), np.int32), [1.0] * R, 10)
    z = np.zeros((1, 4097), np.int32)
    with pytest.raises(_native.NrtGpuUnsupported):
        rescore_combine(gpu_ctx, z, z.astype(np.float32), z.astype(np.uint8), z.astype(np.float32), 1.0, 1.0)


def test_blend_tails_after_a_fuller_call(gpu_ctx):
    rng = np.random.default_rng(9)
    R, nq, top_in, top_out = 2, 5, 300, 500
    docs = np.stack([np.stack([rng.permutation(1000)[:top_in] + 1 for _ in range(nq)]) for _ in range(R)]).astype(np.int32)
    scores = np.sort(rng.random((R, nq, top_in)).astype(np.float32), axis=2)[:, :, ::-1].copy()
    full = np.full((R, nq), top_in, np.int32)
    few = rng.integers(0, 20, (R, nq)).astype(np.int32)
    boosts = [1.0, 0.5]
    for call in (lambda c: blend_rrf(gpu_ctx, docs, c, boosts, 60, top_out),
                 lambda c: blend_scores(gpu_ctx, "max", docs, scores, c, boosts, top_out)):
        d, s, c, t = call(full)
        assert (c >= top_in).all()
        d, s, c, t = call(few)
        assert (c < 40).all()
        for q in range(nq):
            assert not d[q, c[q]:].any() and not s[q, c[q]:].view(np.uint32).any(), q


# ---- end to end: a broad batch, then rare terms with the same nq and k: the second pages' tails must be zero ----

@pytest.fixture(scope="module")
def tail_shard(built):
    from nrtsearch_b200 import index as ix
    from nrtsearch_b200.search import BooleanQuery, Occur, TermQuery
    vocab = 5_000
    sh = ix.synth_text_shard(50_000, vocab)
    sh.term_df = np.diff(sh.term_off).astype(np.int64)
    broad_t = ix.synth_query_terms(32, 2, vocab, seed=11, log10_lo=0.0, log10_hi=1.0)
    rare_t = ix.synth_query_terms(32, 2, vocab, seed=12, log10_lo=3.3, log10_hi=3.7)
    broad = [BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD).add(TermQuery(int(t[1])), Occur.SHOULD) for t in broad_t]
    rare = [BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD if i % 2 else Occur.MUST).add(TermQuery(int(t[1])), Occur.MUST)
            for i, t in enumerate(rare_t)]
    return sh, broad, rare


K_TAIL = 200


def _check_rare(sh, rare, docs, scores, counts, what):
    from nrtsearch_b200.search import compile_queries
    wd, ws, wc, _, _ = oracle.search_compiled(oracle.OracleIndex(sh), *compile_queries(rare), K_TAIL)
    assert (wc < K_TAIL).all() and (wc > 0).any(), "the rare batch must leave short pages"
    _assert_pages(docs, scores, counts, [(wd[q, :wc[q]], ws[q, :wc[q]]) for q in range(len(rare))], what)


def test_index_searcher_tails(gpu_ctx, tail_shard):
    from nrtsearch_b200.search import GpuIndex, GpuIndexSearcher, RelevanceCollector
    sh, broad, rare = tail_shard
    gix = GpuIndex(gpu_ctx, sh)
    try:
        s = GpuIndexSearcher(gix)
        assert (s.search_batch(broad, RelevanceCollector(K_TAIL, INT_MAX)).counts == K_TAIL).all()
        r = s.search_batch(rare, RelevanceCollector(K_TAIL, INT_MAX))
        _check_rare(sh, rare, r.docs, r.scores, r.counts, "GpuIndexSearcher")
    finally:
        gix.close()


def test_leaf_searcher_tails(gpu_ctx, tail_shard):
    from nrtsearch_b200.search import GpuIndex, GpuLeafSearcher, RelevanceCollector
    sh, broad, rare = tail_shard
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in ((0, 20_000), (20_000, 50_000))]
    try:
        s = GpuLeafSearcher(gpu_ctx, leaves)
        assert (s.search_batch(broad, RelevanceCollector(K_TAIL, INT_MAX)).counts == K_TAIL).all()
        r = s.search_batch(rare, RelevanceCollector(K_TAIL, INT_MAX))
        _check_rare(sh, rare, r.docs, r.scores, r.counts, "GpuLeafSearcher")
        s.close()
    finally:
        for l in leaves:
            l.close()


def test_prepared_batch_bound_to_device_buffers(gpu_ctx, tail_shard):
    import torch
    from nrtsearch_b200.search import GpuIndex, GpuIndexSearcher, RelevanceCollector
    sh, broad, rare = tail_shard
    gix = GpuIndex(gpu_ctx, sh)
    dev = torch.device("cuda", 0)
    nq = len(rare)
    try:
        s = GpuIndexSearcher(gix)
        b = s.prepare(rare, RelevanceCollector(K_TAIL, INT_MAX))
        od = torch.full((nq * K_TAIL,), th.SENTINEL, dtype=torch.int32, device=dev)
        os_ = torch.full((nq * K_TAIL,), th.SENTINEL, dtype=torch.int32, device=dev)
        oc = torch.full((nq,), th.SENTINEL, dtype=torch.int32, device=dev)
        b.bind_output(od.data_ptr(), os_.data_ptr(), oc.data_ptr())
        b.run()
        torch.cuda.synchronize()
        _check_rare(sh, rare, od.cpu().numpy().reshape(nq, K_TAIL), os_.cpu().numpy().view(np.float32).reshape(nq, K_TAIL),
                    oc.cpu().numpy(), "bind_output")
        b.close()
    finally:
        gix.close()
