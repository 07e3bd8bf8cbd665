"""Every query engine against the object-level reference (tests/query_reference.py) on generated queries
(tests/query_gen.py): each engine that accepts a query returns the reference's page bit for bit -- docs, score bits,
counts -- with totalHits exact when EQUAL_TO and in (threshold, exact] when GREATER_THAN_OR_EQUAL_TO.

The shard: 1.25M docs (two 1,048,576-doc slices of the window engine, three 524,288-doc slices of the probe kernel), two
text fields (the second without norms) with positions, a term with postings at window, granule and slice edges, a term
with tf >= 255 there and elsewhere, a single- and a multi-valued int column, a SORTED and a SORTED_SET keyword column, and
5% deletes. The engines: search_batch on the probe kernel and forced onto the window engine, search_tree, the second pass
(score_docs / score_docs_tree) on hit lists with matches, non-matches, deleted docs, duplicates and docs outside the leaf,
the collector paths with a MaxCollector, a FilterCollector whose filter is the query, GpuLeafSearcher over random cuts
with a one-doc leaf, prepared batches before and after set_live_docs, and the micro-batcher. searchAfter keys come from
the reference's pages at random ranks, with their score's nextafter in both directions."""
import threading

import numpy as np
import pytest

import plan_harness as ph
import query_gen as qg
from nrtsearch_b200 import _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, FilterCollector, GpuBatcher, GpuIndex, GpuIndexSearcher,
                                   GpuLeafSearcher, MatchAllDocsQuery, MaxCollector, Occur, RelevanceCollector, ScoreDoc,
                                   TermQuery, _resolve_all, compile_queries, compile_tree)
from query_reference import Reference
from test_gpu_tree import N_DOCS, V, two_field_shard
from test_gpu_wide import assert_probe, assert_wide

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
KS = (1, 7, 100, 512, 513, 1024)
KMAX = 1024
SEEDS = (11, 12, 13, 14)
NQ = 64
HITS = 192   # second-pass hit list per query
PROBE_EDGES = [d for e in (1024, 2048, 524_288, 1_048_576, 2 * 524_288 + 1024) for d in (e - 1, e)]


def build_shard():
    """two_field_shard plus: field 1 without norms, term 2V + 1 (field 0) with tf 255..555 at probe edges and random
    docs, an absent term, positions for every posting, and keyword columns"""
    sh = two_field_shard()
    rng = np.random.default_rng(5)
    heavy = np.unique(np.concatenate([PROBE_EDGES, rng.choice(N_DOCS, 40, replace=False)])).astype(np.int32)
    hf = rng.integers(255, 556, len(heavy)).astype(np.int32)
    end = sh.term_off[-1] + len(heavy)
    sh.term_off = np.concatenate([sh.term_off, [end, end]]).astype(np.int64)   # and term 2V + 2 (field 1): no postings
    sh.post_docs = np.concatenate([sh.post_docs, heavy])
    sh.post_freqs = np.concatenate([sh.post_freqs, hf])
    sh.term_field = np.concatenate([sh.term_field, [0, 1]]).astype(np.int32)
    sh.term_df = np.diff(sh.term_off).astype(np.int64)
    sh.fields[0].sum_total_term_freq += int(hf.sum())
    sh.fields[1].norms = None
    # positions: the tokens of each (doc, field) take 0..len-1 in random order
    post_field = np.repeat(sh.term_field, np.diff(sh.term_off)).astype(np.int64)
    key = np.repeat(sh.post_docs.astype(np.int64) * 2 + post_field, sh.post_freqs)
    order = np.lexsort((rng.random(len(key)), key))
    sk = key[order]
    start = np.concatenate([[0], np.nonzero(sk[1:] != sk[:-1])[0] + 1])
    rank = np.arange(len(sk)) - np.repeat(start, np.diff(np.concatenate([start, [len(sk)]])))
    pos = np.empty(len(sk), np.int64)
    pos[order] = rank
    tok_post = np.repeat(np.arange(len(sh.post_docs)), sh.post_freqs)
    sh.post_positions = pos[np.lexsort((pos, tok_post))].astype(np.int32)
    del key, order, sk, rank, pos, tok_post
    words = sorted({"", "a", "ab", "abc", "b", "ba", "café", "cafe", "d\U0001F600"} | {f"k{i:03d}" for i in range(120)})
    terms = [w.encode() for w in words]
    single = rng.integers(-1, len(terms), N_DOCS).astype(np.int32)     # -1: no value
    draw = np.sort(rng.integers(0, len(terms), (N_DOCS, 3)), axis=1)
    keep = (np.arange(3)[None, :] < rng.integers(0, 4, N_DOCS)[:, None])
    keep[:, 1:] &= draw[:, 1:] != draw[:, :-1]
    off = np.zeros(N_DOCS + 1, np.int64)
    np.cumsum(keep.sum(1), out=off[1:])
    sh.keyword_columns = [ix.KeywordColumn(terms, single), ix.KeywordColumn(terms, draw[keep].astype(np.int32), off)]
    return sh


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    sh = build_shard()
    g = GpuIndex(gpu_ctx, sh)
    plane, _ = ph.index_rules(sh.n_docs, sh.term_off)
    df = np.diff(sh.term_off)
    f0 = np.nonzero((sh.term_field == 0) & (df > 0))[0]
    by_df = f0[np.argsort(-df[f0], kind="stable")]
    space = qg.space_of(sh, [(0, False), (1, True)], plane_terms=np.nonzero(plane >= 0)[0][:64],
                        phrase_terms=by_df[20:80])
    space.terms["edge"] = np.array([2 * V], np.int64)
    yield sh, g, space, Reference(sh)
    g.close()


def pad_query(space):
    """five SHOULD terms: a batch holding it runs on the window engine"""
    q = BooleanQuery()
    for t in space.terms["mid"][:5]:
        q.add(TermQuery(int(t)), Occur.SHOULD)
    return q


class Truth:
    """what the reference says of one query: the top KMAX page, totalHits, the max of column 0 over the matches, pages
    after three searchAfter keys, and a hit list with its per-doc match flags and scores"""

    def __init__(self, ref, q, rng, sh):
        p, s = ref.eval(q)
        live = p & ref.live
        m = np.nonzero(live)[0]
        sc = s[m]
        self.docs, self.scores, self.total = ref.page_of(m, sc, KMAX)
        self.col_max = float(sh.columns[0][m].max()) if len(m) else -np.finfo(np.float64).max
        self.after = []
        n = len(self.docs)
        if n:
            r = int(rng.integers(n))
            d, s0 = int(self.docs[r]), np.float32(self.scores[r])
            for a in (s0, np.nextafter(s0, np.float32(np.inf)), np.nextafter(s0, np.float32(-np.inf))):
                sd = ScoreDoc(d, float(a))
                self.after.append((sd, *ref.page_of(m, sc, 100, sd)))
        picks = [rng.choice(m, min(len(m), 90), replace=False) if len(m) else np.zeros(0, np.int64),
                 rng.integers(0, N_DOCS, 60), rng.choice(np.nonzero(~ref.live)[0], 20, replace=False)]
        hits = np.concatenate(picks).astype(np.int64)
        hits = np.concatenate([hits, hits[rng.integers(0, len(hits), 10)], [-1, -7, N_DOCS, N_DOCS + 5, INT_MAX],
                               rng.integers(0, N_DOCS, HITS)])[:HITS]
        self.hits = hits[rng.permutation(HITS)]
        inside = (self.hits >= 0) & (self.hits < N_DOCS)
        loc = np.where(inside, self.hits, 0)
        self.hit_match = inside & live[loc]
        self.hit_score = np.where(self.hit_match, s[loc], np.float32(0)).astype(np.float32)


@pytest.fixture(scope="module", params=SEEDS)
def batch(request, corpus):
    sh, g, space, ref = corpus
    seed = request.param
    queries = qg.Generator(space, seed).queries(NQ)
    rng = np.random.default_rng(seed)
    truths = [Truth(ref, q, rng, sh) for q in queries]
    pad = pad_query(space)
    return seed, queries, truths, Truth(ref, pad, rng, sh), pad


def check(res, truths, queries, rows, k, thr, seed, what):
    for row, i in enumerate(rows):
        t = truths[i]
        n = min(len(t.docs), k)
        msg = f"{what} k={k} thr={thr}: {qg.describe(seed, i, queries[i])}"
        assert int(res.counts[row]) == n, f"{msg}: counts {res.counts[row]} vs {n}"
        assert np.array_equal(res.docs[row, :n], t.docs[:n]), f"{msg}: docs differ"
        assert np.array_equal(res.scores[row, :n].view(np.uint32), t.scores[:n].view(np.uint32)), f"{msg}: scores differ"
        if res.relation[row]:
            assert thr < int(res.total_hits[row]) <= t.total, f"{msg}: totalHits {res.total_hits[row]} of {t.total} (GTE)"
        else:
            assert int(res.total_hits[row]) == t.total, f"{msg}: totalHits {res.total_hits[row]} vs {t.total}"


def tagged(queries, tag):
    return [i for i, q in enumerate(queries) if tag in qg.engines(q)]


def test_generated_batches_cover_the_engines(batch):
    seed, queries, truths, _, _ = batch
    assert len(tagged(queries, "flat_narrow")) >= 8 and len(tagged(queries, "flat_wide")) >= len(tagged(queries, "flat_narrow"))
    totals = np.array([t.total for t in truths])
    assert (totals > 0).mean() > 0.35 and (totals > KMAX).any(), f"seed {seed}: {totals}"


@pytest.mark.parametrize("thr", [INT_MAX, 1000])
def test_search_batch_narrow_and_wide(corpus, batch, thr):
    sh, g, space, _ = corpus
    seed, queries, truths, pad_truth, pad = batch
    s = GpuIndexSearcher(g)
    narrow = tagged(queries, "flat_narrow")
    wide = tagged(queries, "flat_wide")
    qs = [queries[i] for i in narrow]
    assert_probe(g, _resolve_all(qs, g), 100, thr)
    for k in (1, 7, 100, 512):
        check(s.search_batch(qs, RelevanceCollector(k, thr)), truths, queries, narrow, k, thr, seed, "probe")
    tw = truths + [pad_truth]
    qw, rows = [queries[i] for i in wide] + [pad], wide + [len(queries)]
    assert_wide(g, _resolve_all(qw, g), 100, thr)
    for k in KS:
        check(s.search_batch(qw, RelevanceCollector(k, thr)), tw, queries + [pad], rows, k, thr, seed, "window, flat")


@pytest.mark.parametrize("thr", [INT_MAX, 1000])
def test_search_tree(corpus, batch, thr):
    _, g, _, _ = corpus
    seed, queries, truths, _, _ = batch
    s = GpuIndexSearcher(g)
    for k in KS:
        check(s.search_tree(queries, RelevanceCollector(k, thr)), truths, queries, range(len(queries)), k, thr, seed, "tree")


def test_search_after(corpus, batch):
    _, g, _, _ = corpus
    seed, queries, truths, _, _ = batch
    s = GpuIndexSearcher(g)
    rows = [i for i, t in enumerate(truths) if t.after]
    narrow = [i for i in tagged(queries, "flat_narrow") if truths[i].after]
    for v in range(3):   # the page's own key, nextafter up, nextafter down
        after = [truths[i].after[v][0] for i in rows]
        res = s.search_tree([queries[i] for i in rows], RelevanceCollector(100, INT_MAX), search_after=after)
        res_n = s.search_batch([queries[i] for i in narrow], RelevanceCollector(100, INT_MAX),
                               search_after=[truths[i].after[v][0] for i in narrow])
        for res_, rows_, what in ((res, rows, "tree"), (res_n, narrow, "probe")):
            for row, i in enumerate(rows_):
                sd, d, sc, total = truths[i].after[v]
                msg = f"{what} after {sd} (variant {v}): {qg.describe(seed, i, queries[i])}"
                assert int(res_.counts[row]) == len(d), f"{msg}: counts {res_.counts[row]} vs {len(d)}"
                assert np.array_equal(res_.docs[row, :len(d)], d), f"{msg}: docs differ"
                assert np.array_equal(res_.scores[row, :len(d)].view(np.uint32), sc.view(np.uint32)), f"{msg}: scores"
                assert int(res_.total_hits[row]) == total, f"{msg}: totalHits"


def test_second_pass(corpus, batch):
    _, g, _, _ = corpus
    seed, queries, truths, _, _ = batch
    s = GpuIndexSearcher(g)
    for what, rows, fn in (("score_docs", tagged(queries, "flat_wide"), s.score_docs),
                           ("score_docs_tree", list(range(len(queries))), s.score_docs_tree)):
        hits = np.stack([truths[i].hits for i in rows]).astype(np.int32)
        m, sc = fn([queries[i] for i in rows], hits)
        for row, i in enumerate(rows):
            msg = f"{what}: {qg.describe(seed, i, queries[i])}"
            assert np.array_equal(m[row] != 0, truths[i].hit_match), f"{msg}: match flags differ"
            assert np.array_equal(sc[row].view(np.uint32), truths[i].hit_score.view(np.uint32)), f"{msg}: scores differ"


def test_collectors(corpus, batch):
    _, g, _, _ = corpus
    seed, queries, truths, _, _ = batch
    s = GpuIndexSearcher(g)
    narrow = tagged(queries, "flat_narrow")
    for what, rows, fn, ks in (("search_with_collectors", narrow, s.search_with_collectors, (7, 512)),
                               ("search_tree_with_collectors", list(range(len(queries))), s.search_tree_with_collectors,
                                (7, 1024))):
        for k in ks:
            res, outs = fn([queries[i] for i in rows], RelevanceCollector(k, INT_MAX), [MaxCollector(0, "int")])
            check(res, truths, queries, rows, k, INT_MAX, seed, what)
            want = np.array([truths[i].col_max for i in rows])
            assert np.array_equal(outs[0], want), f"{what} seed {seed}: max over the matches"
    # the query as a FilterCollector's filter under match-all: docCount = its live matches
    outs = []
    for c in range(0, len(narrow), 4):   # four filters (eight aggregations) per search
        fc = [FilterCollector(queries[i], (("max", MaxCollector(0, "int")),)) for i in narrow[c:c + 4]]
        outs += s.search_with_collectors([MatchAllDocsQuery()], RelevanceCollector(1, INT_MAX), fc)[1]
    for j, i in enumerate(narrow):
        msg = f"filter collector: {qg.describe(seed, i, queries[i])}"
        assert int(outs[j]["doc_count"][0]) == truths[i].total, msg
        assert float(outs[j]["max"][0]) == truths[i].col_max, msg


def test_leaf_searcher(gpu_ctx, corpus, batch):
    sh, _, _, _ = corpus
    seed, queries, truths, _, _ = batch
    rng = np.random.default_rng(seed)
    one = int(rng.integers(1, N_DOCS - 1))
    cuts = sorted({0, one, one + 1, int(rng.integers(1, N_DOCS)), int(rng.integers(1, N_DOCS)), N_DOCS})
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    try:
        ls = GpuLeafSearcher(gpu_ctx, leaves)
        narrow = tagged(queries, "flat_narrow")
        for k in (7, 100):
            check(ls.search_batch([queries[i] for i in narrow], RelevanceCollector(k, INT_MAX)), truths, queries, narrow, k,
                  INT_MAX, seed, f"leaves {cuts}")
            check(ls.search_tree(queries, RelevanceCollector(k, INT_MAX)), truths, queries, range(len(queries)), k, INT_MAX,
                  seed, f"leaves {cuts}, tree")
        ls.close()
    finally:
        for g in leaves:
            g.close()


def test_prepared_batches_follow_live_docs(corpus, batch):
    sh, g, _, _ = corpus
    seed, queries, truths, _, _ = batch
    s = GpuIndexSearcher(g)
    rows = list(range(0, len(queries), 2))
    flat = [i for i in tagged(queries, "flat_narrow")]
    rng = np.random.default_rng(seed + 100)
    live2 = (sh.live_docs != 0) & (rng.random(N_DOCS) > 0.03)
    ref2 = Reference(ix.HostShard(**{**sh.__dict__, "live_docs": live2.astype(np.uint8)}))
    after = {i: Truth(ref2, queries[i], np.random.default_rng(0), sh) for i in sorted(set(rows) | set(flat))}
    k = 100
    bt = s.prepare_tree([queries[i] for i in rows], RelevanceCollector(k, INT_MAX))
    bf = s.prepare([queries[i] for i in flat], RelevanceCollector(k, INT_MAX))
    try:
        for b, rs, what in ((bt, rows, "prepared tree"), (bf, flat, "prepared flat")):
            b.run()
            check(b.fetch(), truths, queries, rs, k, INT_MAX, seed, what)
        g.set_live_docs(live2.astype(np.uint8))
        for b, rs, what in ((bt, rows, "prepared tree"), (bf, flat, "prepared flat")):
            b.run()
            check(b.fetch(), after, queries, rs, k, INT_MAX, seed, what + " after set_live_docs")
    finally:
        g.set_live_docs(sh.live_docs)
        bt.close()
        bf.close()


def test_micro_batcher(corpus, batch):
    _, g, _, _ = corpus
    seed, queries, truths, _, _ = batch
    rows = tagged(queries, "flat_wide")
    b = GpuBatcher(g, max_batch=32, max_wait_us=20_000)
    results = {}

    def worker(i):
        results[i] = b.submit(queries[i], RelevanceCollector(100, INT_MAX))
    ts = [threading.Thread(target=worker, args=(i,)) for i in rows]
    [t.start() for t in ts]
    [t.join() for t in ts]
    b.close()
    for i in rows:
        td, _ = results[i]
        t = truths[i]
        n = min(len(t.docs), 100)
        msg = f"batcher: {qg.describe(seed, i, queries[i])}"
        assert [sd.doc for sd in td.score_docs] == t.docs[:n].tolist(), msg
        assert np.array_equal(np.array([sd.score for sd in td.score_docs], np.float32).view(np.uint32), t.scores[:n].view(np.uint32)), msg
        assert td.total_hits.value == t.total, msg


# ---------------------------------------------------------------- non-finite boosts

def test_non_finite_boosts_are_refused_and_write_nothing(corpus):
    _, g, _, _ = corpus
    s = GpuIndexSearcher(g)
    lib = _native.gpu_lib()
    for b in (float("nan"), float("inf")):
        bad = [BooleanQuery().add(TermQuery(1), Occur.SHOULD).add(BoostQuery(TermQuery(2), b), Occur.SHOULD)]
        for call in (lambda: s.search_batch(bad, RelevanceCollector(10, INT_MAX)), lambda: s.search_tree(bad, RelevanceCollector(10, INT_MAX)),
                     lambda: s.score_docs(bad, np.zeros((1, 4), np.int32)), lambda: s.score_docs_tree(bad, np.zeros((1, 4), np.int32)),
                     lambda: s.prepare(bad, RelevanceCollector(10, INT_MAX)), lambda: s.prepare_tree(bad, RelevanceCollector(10, INT_MAX)),
                     lambda: s.search_with_collectors(bad, RelevanceCollector(10, INT_MAX), [MaxCollector(0, "int")]),
                     lambda: s.search_tree_with_collectors(bad, RelevanceCollector(10, INT_MAX), [MaxCollector(0, "int")])):
            with pytest.raises(ValueError, match="Boost must be a finite number"):
                call()
        # the C ABI, past the Python compilers: NRTGPU_ERR_INVALID and the output buffers untouched
        good = [BooleanQuery().add(TermQuery(1), Occur.SHOULD).add(TermQuery(2), Occur.SHOULD)]
        for arrays in (compile_queries(good), compile_tree(good)):
            carr = arrays[0]
            carr[1].boost = b
            out = [np.full(10, 77, np.int32), np.full(10, 7.5, np.float32), np.full(1, 77, np.int32), np.full(1, 77, np.int64),
                   np.full(1, 77, np.uint8), np.full(1, 77, np.uint8), np.full(1, 77, np.uint8)]
            if len(arrays) == 4:
                rc = lib.nrtgpu_search_bool(g.handle, carr, arrays[1], arrays[2], arrays[3], 10, INT_MAX, 0, None,
                                            *[o.ctypes.data for o in out[:5]])
            else:
                rc = lib.nrtgpu_search_tree(g.handle, carr, arrays[1], arrays[2], arrays[3], arrays[4], arrays[5], 10, INT_MAX, 0,
                                            None, None, *[o.ctypes.data for o in out])
            assert rc == 1 and "Boost must be a finite number" in lib.nrtgpu_last_error().decode()
            for o, v in zip(out, (77, 7.5, 77, 77, 77, 77, 77)):
                assert (o == v).all(), "a refused call wrote output"
    with pytest.raises(ValueError, match="Boost must be a finite number"):
        b = GpuBatcher(g, max_batch=4, max_wait_us=100)
        try:
            b.submit(BoostQuery(TermQuery(1), float("nan")), RelevanceCollector(10, INT_MAX))
        finally:
            b.close()
