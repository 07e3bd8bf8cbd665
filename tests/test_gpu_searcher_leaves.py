"""Searchers over several leaves (nrtgpu_searcher_*): sorted search, query trees and phrases, and kNN, every leaf searched
into a device record and the records merged on the device. Checked bit for bit against the whole shard's references
(sort_fields_reference, phrase_reference / tree_reference, oracle.knn_exact) and against the single-image search of the
whole shard; the sorted merge kernel (nrtgpu_merge_sorted_packed) alone against a numpy lexsort of crafted records."""
import ctypes as C
import zlib

import numpy as np
import pytest

import oracle
import phrase_reference as pr
import searcher_leaves as sl
import sort_single_shard as ss
from helpers import assert_same_hits
from nrtsearch_b200 import NrtGpuError, _native
from nrtsearch_b200._native import CollectionTimeoutException, SearchLimits
from nrtsearch_b200.index import HostShard
from nrtsearch_b200.search import (BooleanQuery, DisjunctionMaxQuery, FieldDoc, GpuIndex, GpuIndexSearcher, GpuLeafSearcher, Occur,
                                   PhraseQuery, RangeQuery, RelevanceCollector, ScoreDoc, SortFieldCollector, SortType, TermQuery,
                                   compile_queries)
from nrtsearch_b200.shards import SortedPackedGather, unpack_sorted_record

pytestmark = pytest.mark.gpu
INVALID = 1
INT_MAX = 2**31 - 1
I64_MIN, I64_MAX = -2**63, 2**63 - 1
COLUMN, DOCID, SCORE = 1, 2, 3


# ---------------------------------------------------------------- the merge kernel alone

def _f32_bits(x):
    return np.asarray(x, np.float32).view(np.uint32).astype(np.int64)


VALUE_POOL = np.array([I64_MIN, I64_MAX, 0, -1, 1, 7, 7, 7,
                       ss._sortable_f64(np.nan), ss._sortable_f64(-0.0), ss._sortable_f64(0.0), ss._sortable_f64(np.inf),
                       ss._sortable_f64(-np.inf), ss._sortable_f32(np.nan), ss._sortable_f32(-0.0), ss._sortable_f32(np.inf)],
                      np.int64)
SCORE_POOL = _f32_bits([0.0, -0.0, 1.5, 1.5, 1.5, 2.25, 3.0e-39, 7.0, np.inf])


def craft(rng, fields, n_lists, nq, k, equal=False):
    """n_lists records of nq queries: each (list, query) a page of 0..k entries sorted under `fields`, global docs distinct"""
    nf = len(fields)
    words = sl_words(nq, k, nf)
    recs = np.zeros((n_lists, words), np.int32)
    ne = sl.ref.deciding(fields)
    for l in range(n_lists):
        r = recs[l]
        docs, vals, counts, flags, tot = unpack_sorted_record(r, nq, k, nf)
        counts[:] = rng.integers(0, k + 1, nq)
        if n_lists > 1:
            counts[rng.random(nq) < 0.15] = 0
        flags[:] = rng.integers(0, 8, nq) * (rng.random(nq) < 0.3)
        tot[:] = counts + rng.integers(0, 1 << 40, nq)
        for q in range(nq):
            c = int(counts[q])
            d = np.sort(rng.choice(1 << 20, c, replace=False)) * n_lists + l    # distinct across lists
            v = np.zeros((c, nf), np.int64)
            for j, f in enumerate(fields):
                if f[0] == SCORE:
                    v[:, j] = SCORE_POOL[rng.integers(0, 2 if equal else len(SCORE_POOL), c)]
                elif f[0] == DOCID:
                    v[:, j] = d + 1000 * j
                else:
                    v[:, j] = VALUE_POOL[rng.integers(0, 1 if equal else len(VALUE_POOL), c)]
            keys = [sl.ref.field_keys(f, v[:, j]) for j, f in enumerate(fields[:ne])]
            o = np.lexsort([d] + list(reversed(keys)))
            docs[q, :c] = d[o]
            vals[q, :c] = v[o]
    return recs


def sl_words(nq, k, nf):
    return int(_native.gpu_lib().nrtgpu_sorted_packed_words(nq, k, nf))


def run_merge(gpu_ctx, fields, recs, nq, k):
    import torch
    nf = len(fields)
    words = sl_words(nq, k, nf)
    dev = torch.device("cuda", 0)
    d_in = torch.from_numpy(recs.reshape(-1)).to(dev)
    d_out = torch.full((words,), -7, dtype=torch.int32, device=dev)
    arr = (_native.SortField * nf)(*[_native.SortField(*f) for f in fields])
    _native.check(_native.gpu_lib().nrtgpu_merge_sorted_packed(gpu_ctx.handle, arr, nf, len(recs), nq, k, d_in.data_ptr(),
                                                               d_out.data_ptr(), None))
    torch.cuda.synchronize()
    return d_out.cpu().numpy()


def check_merge(fields, recs, out, nq, k):
    nf = len(fields)
    lists = [unpack_sorted_record(r, nq, k, nf) for r in recs]
    docs, vals, counts, flags, tot = unpack_sorted_record(out, nq, k, nf)
    assert np.array_equal(tot, sum(x[4] for x in lists))
    assert np.array_equal(flags, np.bitwise_or.reduce([x[3] for x in lists]))
    for q in range(nq):
        md, mv = sl.merge_sorted(fields, [(x[0][q], x[1][q], x[2][q]) for x in lists], k)
        assert counts[q] == len(md), q
        assert np.array_equal(docs[q, :len(md)], md) and np.array_equal(vals[q, :len(md)], mv), q
        assert not docs[q, len(md):].any() and not vals[q, len(md):].any(), q


MERGE_FIELDS = {
    "col": [(COLUMN, 0, 0, 0, 0)],
    "col-rev": [(COLUMN, 0, 1, 0, 0)],
    "docid-rev": [(DOCID, 0, 1, 0, 0)],
    "score": [(SCORE, 0, 0, 0, 0)],
    "score-rev,col": [(SCORE, 0, 1, 0, 0), (COLUMN, 0, 0, 0, 0)],
    "score,col-rev,col": [(SCORE, 0, 0, 0, 0), (COLUMN, 0, 1, 0, 0), (COLUMN, 1, 0, 0, 0)],
    "col,docid,col": [(COLUMN, 0, 0, 0, 0), (DOCID, 0, 0, 0, 0), (COLUMN, 1, 1, 0, 0)],
    "8 mixed": [(COLUMN, i, i % 2, 0, 0) for i in range(7)] + [(DOCID, 0, 1, 0, 0)],
    "8 columns": [(COLUMN, i, (i + 1) % 2, 0, 0) for i in range(8)],
}


@pytest.mark.parametrize("name", list(MERGE_FIELDS))
@pytest.mark.parametrize("n_lists,k", [(1, 40), (2, 1), (2, 1024), (7, 40), (64, 40), (64, 1024)])
def test_merge_kernel(gpu_ctx, name, n_lists, k):
    fields = MERGE_FIELDS[name]
    nq = 3 if k == 1024 else 24
    rng = np.random.default_rng(zlib.crc32(f"{name}/{n_lists}/{k}".encode()))
    recs = craft(rng, fields, n_lists, nq, k)
    check_merge(fields, recs, run_merge(gpu_ctx, fields, recs, nq, k), nq, k)


@pytest.mark.parametrize("name", ["col", "score", "8 mixed", "8 columns"])
def test_merge_kernel_ties_decided_by_doc(gpu_ctx, name):
    fields, nq, k = MERGE_FIELDS[name], 16, 40
    recs = craft(np.random.default_rng(5), fields, 7, nq, k, equal=True)
    check_merge(fields, recs, run_merge(gpu_ctx, fields, recs, nq, k), nq, k)


def test_merge_kernel_many_queries(gpu_ctx):
    fields, nq, k = MERGE_FIELDS["score-rev,col"], 1100, 40
    recs = craft(np.random.default_rng(9), fields, 7, nq, k)
    check_merge(fields, recs, run_merge(gpu_ctx, fields, recs, nq, k), nq, k)


def test_merge_kernel_refusals(gpu_ctx):
    lib = _native.gpu_lib()
    arr = (_native.SortField * 9)(*[_native.SortField(1, 0, 0, 0, 0)] * 9)
    for n_fields, n_lists in ((0, 2), (9, 2), (1, 0)):
        assert lib.nrtgpu_merge_sorted_packed(gpu_ctx.handle, arr, n_fields, n_lists, 4, 4, C.c_void_p(8), C.c_void_p(8), None) == INVALID


# ---------------------------------------------------------------- sorted search over leaves

@pytest.fixture(scope="module")
def sorted_setup(gpu_ctx):
    sh = ss.make_shard(sl.N, sl.DOC_BASE, sl.TIE_LO)
    cuts = sl.cuts()
    whole = GpuIndex(gpu_ctx, sh)
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    s = GpuLeafSearcher(gpu_ctx, leaves)
    yield sh, oracle.OracleIndex(sh), whole, leaves, s
    s.close()
    for g in leaves + [whole]:
        g.close()


def as_fields(res, nf):
    return res.sort_values.reshape(res.counts.shape[0], -1, nf)


def assert_sorted_equal(res, w, what, nf):
    wd, wv, wc, wt = w
    assert np.array_equal(res.counts, wc), what
    assert np.array_equal(res.total_hits, wt) and not res.relation.any(), what
    v = as_fields(res, nf)
    for q in range(len(wc)):
        n = wc[q]
        assert np.array_equal(res.docs[q, :n], wd[q, :n]), (what, q)
        assert np.array_equal(v[q, :n], wv[q, :n]), (what, q)


@pytest.mark.parametrize("sid,fields", sl.all_sorts(), ids=[s for s, _ in sl.all_sorts()])
def test_sorted_search_over_leaves(sorted_setup, sid, fields):
    sh, oix, whole, _, s = sorted_setup
    nf = len(fields)
    sort = fields[0] if nf == 1 and fields[0].field not in ("score", ss.C_MV) else fields   # one image: a multi-valued column
    for k in (1, 40, 512):
        res = s.search_sorted(ss.QUERIES, SortFieldCollector(k, sort))
        one = GpuIndexSearcher(whole).search_sorted(ss.QUERIES, SortFieldCollector(k, sort))
        assert res.sort_values.shape == one.sort_values.shape
        w = sl.reference(sh, ss.QUERIES, k, fields, oix=oix)
        assert_sorted_equal(res, w, f"{sid} k={k} reference", nf)
        assert_sorted_equal(res, (one.docs, as_fields(one, nf), one.counts, one.total_hits), f"{sid} k={k} single image", nf)
        assert not res.hit_timeout.any() and not res.terminated_early.any()


@pytest.mark.parametrize("sid", ["c0int-asc-last", "c4double-desc-first", "docid-desc", "score,mv-max,i64", "8 fields",
                                 "one,f32-desc-last,docid"])
def test_paging_across_leaves(sorted_setup, sid):
    """pages of 40, each after the last FieldDoc of the previous one, concatenate to the reference's complete list"""
    sh, oix, _, _, s = sorted_setup
    fields = dict(sl.all_sorts())[sid]
    nf = len(fields)
    full = sl.reference(sh, ss.QUERIES, 4000, fields, oix=oix)
    qids = [q for q in range(len(ss.QUERIES)) if 0 < full[3][q] <= 4000][:5]
    assert len(qids) >= 3
    got = {q: [] for q in qids}
    after = {q: None for q in qids}
    active = list(qids)
    while active:
        aft = [after[q] for q in active]
        res = s.search_sorted([ss.QUERIES[q] for q in active], SortFieldCollector(40, fields),
                              None if all(a is None for a in aft) else aft)
        nxt = []
        for i, q in enumerate(active):
            n = int(res.counts[i])
            assert res.total_hits[i] == full[3][q]
            got[q].extend((int(res.docs[i, j]), tuple(int(x) for x in res.sort_values[i, j])) for j in range(n))
            if n == 40 and len(got[q]) < full[3][q]:
                after[q] = FieldDoc(int(res.docs[i, n - 1]), 0, tuple(int(x) for x in res.sort_values[i, n - 1]))
                nxt.append(q)
        active = nxt
    for q in qids:
        c = int(full[2][q])
        assert [d for d, _ in got[q]] == full[0][q, :c].tolist(), (sid, q)
        assert [v for _, v in got[q]] == [tuple(x) for x in full[1][q, :c].tolist()], (sid, q)


def test_two_shards_sorted_packed_merge(gpu_ctx, sorted_setup):
    """nrtgpu_search_sorted_fields_packed per doc-range shard, then the sorted PackedGather merge on the device"""
    import torch
    sh, oix, _, _, _ = sorted_setup
    shards = [GpuIndex(gpu_ctx, sh.doc_range(0, 250_000)), GpuIndex(gpu_ctx, sh.doc_range(250_000, sl.N))]
    dev = torch.device("cuda", 0)
    lib = _native.gpu_lib()
    try:
        for sid in ("c2long-desc-last", "score,mv-max,i64", "8 fields"):
            fields = dict(sl.all_sorts())[sid]
            k, nq = 40, len(ss.QUERIES)
            pg = SortedPackedGather(nq, k, fields, 2, dev)
            carr, ncl, qarr, _ = compile_queries(ss.QUERIES)
            for g, part in zip(shards, pg.all.view(2, pg.words)):
                _native.check(lib.nrtgpu_search_sorted_fields_packed(g.handle, g.sort_order(fields), carr, ncl, qarr, nq, k, 0, None,
                                                                      None, None, part.data_ptr()))
            pg.merge_on_device(gpu_ctx, 0)
            torch.cuda.synchronize()
            d, v, c, flags, tot = pg.unpack()
            wd, wv, wc, wt = sl.reference(sh, ss.QUERIES, k, fields, oix=oix)
            assert np.array_equal(c, wc) and np.array_equal(tot, wt) and not flags.any(), sid
            for q in range(nq):
                assert np.array_equal(d[q, :wc[q]], wd[q, :wc[q]]) and np.array_equal(v[q, :wc[q]], wv[q, :wc[q]]), (sid, q)
    finally:
        for g in shards:
            g.close()


def raw_sorted(s, fields, qs, k, lim, orders=None):
    carr, ncl, qarr, nq = compile_queries(qs)
    orders = [l.sort_order(fields) for l in s.leaves] if orders is None else orders
    arr = (C.c_void_p * max(len(orders), 1))(*[o.value for o in orders])
    out = [np.zeros((nq, k), np.int32), np.zeros((nq, k, len(fields)), np.int64), np.zeros(nq, np.int32), np.zeros(nq, np.int64),
           np.zeros(nq, np.uint8), np.zeros(nq, np.uint8), np.zeros(nq, np.uint8)]
    rc = _native.gpu_lib().nrtgpu_searcher_search_sorted_fields(s.handle, arr, len(orders), carr, ncl, qarr, nq, k, 0, None,
                                                                None if lim is None else C.byref(lim), None,
                                                                *[a.ctypes.data for a in out])
    return rc, out


def test_sorted_refusals_and_limits(gpu_ctx, sorted_setup):
    sh, oix, whole, leaves, s = sorted_setup
    a, b = [SortType(ss.C_I32, field_type="int")], [SortType(ss.C_I32, True, field_type="int")]
    good = [l.sort_order(a) for l in leaves]
    mixed = good[:-1] + [leaves[-1].sort_order(b)]
    other = good[:-1] + [leaves[0].sort_order(a)]
    for orders in (mixed, other, good[:-1]):
        rc, out = raw_sorted(s, a, ss.QUERIES, 10, None, orders)
        assert rc == INVALID and not out[2].any()
    with pytest.raises(NrtGpuError) as e:   # SCORE after the first position keeps its single-image refusal
        s.search_sorted(ss.QUERIES, SortFieldCollector(10, [SortType("score"), SortType("score")]))
    assert e.value.status == 3
    # a deadline already spent: every leaf skips its work items, the merged queries report hit_timeout and relation GTE
    rc, out = raw_sorted(s, a, ss.QUERIES, 10, SearchLimits(1.0, 2.0, 0, 0, 0))
    assert rc == 0
    to, rel = out[5], out[4]
    assert to.any() and rel[to == 1].all()
    rc, _ = raw_sorted(s, a, ss.QUERIES, 10, SearchLimits(1.0, 2.0, 1, 0, 0))
    assert rc == 5
    # terminateAfter: terminated early, relation GTE and the capped count, as on one image
    rc, out = raw_sorted(s, a, [ss.QUERIES[ss.MATCH_ALL]], 10, SearchLimits(0.0, 0.0, 0, 1000, 0))
    assert rc == 0 and out[6][0] == 1 and out[4][0] == 1 and out[3][0] >= 1000


# ---------------------------------------------------------------- trees and phrases over leaves

@pytest.fixture(scope="module")
def phrase_setup(gpu_ctx):
    n = 400_000
    rng = np.random.default_rng(17)
    vocab = 300
    lens = 3 + rng.poisson(7.0, n)
    start = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=start[1:])
    w = 1.0 / np.arange(1, vocab + 1) ** 1.1
    tok = np.searchsorted(np.cumsum(w) / w.sum(), rng.random(int(start[-1]))).astype(np.int64)
    doc = np.repeat(np.arange(n), lens)
    pos = np.arange(int(start[-1])) - start[doc]
    sh = pr.shard_from_token_arrays(n, np.zeros(vocab, np.int32), 1, doc, tok, pos,
                                    live_docs=(rng.random(n) > 0.08).astype(np.uint8))
    sh.columns = [rng.integers(0, 1000, n).astype(np.int64)]
    sh.column_has = [None]
    cuts = [0, 130_000, 130_041, 290_000, n]
    whole = GpuIndex(gpu_ctx, sh)
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    s = GpuLeafSearcher(gpu_ctx, leaves)
    yield sh, whole, leaves, s
    s.close()
    for g in leaves + [whole]:
        g.close()


def T(t):
    return TermQuery(int(t))


def tree_queries():
    S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
    qs = [PhraseQuery([0, 1]), PhraseQuery([2, 0, 5]), PhraseQuery([1, 3], slop=2), PhraseQuery([4, 4], slop=0),
          BooleanQuery().add(PhraseQuery([0, 2]), M).add(T(7), S),
          BooleanQuery().add(PhraseQuery([3, 1], slop=1), S).add(T(40), S).add(RangeQuery(0, 100, 600), F),
          DisjunctionMaxQuery([T(9), T(12), PhraseQuery([0, 3])], 0.3),
          BooleanQuery().add(DisjunctionMaxQuery([T(2), T(8)], 0.1), M).add(BooleanQuery().add(T(30), S).add(T(31), S), S)
          .add(T(5), N),
          BooleanQuery().add(T(250), M).add(T(251), M),
          PhraseQuery([299, 298, 297])]
    return qs


def test_trees_and_phrases_over_leaves(phrase_setup):
    sh, whole, _, s = phrase_setup
    qs = tree_queries()
    oix = oracle.OracleIndex(sh)
    for k, thr in ((1, INT_MAX), (40, INT_MAX), (100, 1000), (1024, INT_MAX)):
        res = s.search_tree(qs, RelevanceCollector(k, thr))
        got = (res.docs, res.scores, res.counts, res.total_hits, res.relation)
        w = pr.search(sh, qs, k, oix=oix)
        assert_same_hits(got, w, check_total=False, what=f"k={k} thr={thr} reference")
        eq = res.relation == 0
        assert np.array_equal(res.total_hits[eq], w[3][eq])
        if thr == INT_MAX:
            assert not res.relation.any()
        one = GpuIndexSearcher(whole).search_tree(qs, RelevanceCollector(k, thr))
        assert_same_hits(got, (one.docs, one.scores, one.counts, one.total_hits, one.relation), check_total=False,
                         what=f"k={k} thr={thr} single image")


def test_trees_search_after_and_limits_over_leaves(phrase_setup):
    sh, whole, leaves, s = phrase_setup
    qs = tree_queries()
    first = s.search_tree(qs, RelevanceCollector(20))
    after = [ScoreDoc(int(first.docs[q, 19]), float(first.scores[q, 19])) if first.counts[q] == 20 else None for q in range(len(qs))]
    res = s.search_tree(qs, RelevanceCollector(20), search_after=after)
    w = pr.search(sh, qs, 20, search_after=after)
    assert_same_hits((res.docs, res.scores, res.counts, res.total_hits, res.relation), w, what="searchAfter")
    # a deadline already spent, on flat queries (the posting-probe kernel honours the deadline)
    flat = [BooleanQuery().add(T(3), Occur.SHOULD).add(T(40), Occur.SHOULD), BooleanQuery().add(T(1), Occur.MUST).add(T(2), Occur.MUST)]
    res = s.search_tree(flat, RelevanceCollector(10, timeout_sec=1.0, elapsed_sec=2.0))
    assert res.hit_timeout.all() and res.relation.all()
    with pytest.raises(CollectionTimeoutException):
        s.search_tree(flat, RelevanceCollector(10, timeout_sec=1.0, elapsed_sec=2.0, disallow_partial_results=True))


def test_phrase_on_a_leaf_without_positions(gpu_ctx, phrase_setup):
    sh, _, leaves, _ = phrase_setup
    bare = sh.doc_range(290_000, 400_000)
    bare.post_positions = None
    g = GpuIndex(gpu_ctx, bare)
    s = GpuLeafSearcher(gpu_ctx, leaves[:3] + [g])
    try:
        with pytest.raises(NrtGpuError) as e:
            s.search_tree([PhraseQuery([0, 1])], RelevanceCollector(10))
        assert e.value.status == INVALID and "position" in e.value.message
        s.search_tree([T(3)], RelevanceCollector(10))   # a tree without phrases still runs
    finally:
        s.close()
        g.close()


# ---------------------------------------------------------------- kNN over leaves

@pytest.fixture(scope="module")
def knn_setup(gpu_ctx):
    n, dims = 60_000, 64
    rng = np.random.default_rng(3)
    corpus = rng.standard_normal((n, dims)).astype(np.float32)
    no_vec = (20_000, 27_000)                                        # the docs of leaf 1 have no vectors
    has = np.ones(n, bool)
    has[no_vec[0]:no_vec[1]] = False
    vdocs = np.nonzero(has)[0].astype(np.int32)
    live = (rng.random(n) > 0.08).astype(np.uint8)
    sim = 0   # L2
    wsh = HostShard(n_docs=n, doc_base=0, term_off=np.zeros(1, np.int64), post_docs=np.zeros(0, np.int32),
                    post_freqs=np.zeros(0, np.int32), fields=[], vectors=np.ascontiguousarray(corpus[vdocs]), vec_similarity=sim,
                    vec_docs=vdocs, live_docs=live)
    wsh.columns = [rng.integers(0, 100, n).astype(np.int64)]
    wsh.column_has = [None]
    cuts = [0, no_vec[0], no_vec[1], 41_000, n]
    leaf_sh = []
    for a, b in zip(cuts, cuts[1:]):
        l = wsh.doc_range(a, b)
        if l.vectors is not None and len(l.vectors) == 0:
            l.vectors, l.vec_docs = None, None
        leaf_sh.append(l)
    whole = GpuIndex(gpu_ctx, wsh)
    leaves = [GpuIndex(gpu_ctx, l) for l in leaf_sh]
    s = GpuLeafSearcher(gpu_ctx, leaves)
    yield corpus, has, live, sim, whole, leaves, s, wsh.columns[0]
    s.close()
    for g in leaves + [whole]:
        g.close()


def test_knn_over_leaves(knn_setup):
    corpus, has, live, sim, whole, leaves, s, _ = knn_setup
    rng = np.random.default_rng(11)
    nq, k = 48, 30
    q = rng.standard_normal((nq, corpus.shape[1])).astype(np.float32)
    boosts = rng.uniform(0.5, 2.0, nq).astype(np.float32)
    filt = (rng.random(len(has)) < 0.3).astype(np.uint8)
    for b, f in ((None, None), (boosts, None), (boosts, filt)):
        d, sc, c = s.knn(q, k, b, f)
        eligible = has.astype(np.uint8) if f is None else (has & (f != 0)).astype(np.uint8)
        wd, ws, wc = oracle.knn_exact(corpus, sim, q, k, filter_docs=eligible, boosts=b, live_docs=live)
        assert np.array_equal(c, wc) and np.array_equal(d, wd)
        od, osc, oc = GpuIndexSearcher(whole).knn(q, k, b, f)
        assert np.array_equal(oc, c) and np.array_equal(od, d)
        assert np.array_equal(osc.view(np.uint32), sc.view(np.uint32))


def test_knn_filtered_over_leaves(knn_setup):
    corpus, has, live, sim, whole, leaves, s, col = knn_setup
    rng = np.random.default_rng(12)
    nq, k = 32, 20
    q = rng.standard_normal((nq, corpus.shape[1])).astype(np.float32)
    ranges = [None, (0, 40), (3, 3), (1, 0)]                         # (1, 0): an empty BooleanQuery matches nothing
    fq = [None if r is None else BooleanQuery() if r == (1, 0) else RangeQuery(0, *r) for r in ranges] * (nq // 4)
    d, sc, c = s.knn(q, k, None, filter_queries=fq)
    od, osc, oc = GpuIndexSearcher(whole).knn(q, k, None, filter_queries=fq)
    assert np.array_equal(oc, c)
    for i in range(nq):   # the page of each query (slots past its count are unspecified)
        n = c[i]
        assert np.array_equal(od[i, :n], d[i, :n]) and np.array_equal(osc[i, :n].view(np.uint32), sc[i, :n].view(np.uint32)), i
    for i in range(nq):
        r = ranges[i % 4]
        elig = has if r is None else has & (col >= r[0]) & (col <= r[1])
        wd, _, wc = oracle.knn_exact(corpus, sim, q[i:i + 1], k, filter_docs=elig.astype(np.uint8), live_docs=live)
        assert c[i] == wc[0] and np.array_equal(d[i, :c[i]], wd[0, :wc[0]]), i


def test_knn_refusals(gpu_ctx, knn_setup):
    _, _, _, _, _, leaves, s, _ = knn_setup
    q = np.zeros((2, 64), np.float32)
    with pytest.raises(NrtGpuError):
        s.knn(q, 0)
    bare = GpuLeafSearcher(gpu_ctx, [leaves[1]])   # no leaf has vectors
    try:
        with pytest.raises(NrtGpuError) as e:
            bare.knn(q, 5)
        assert e.value.status == INVALID
    finally:
        bare.close()
