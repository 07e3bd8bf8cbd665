"""ConstantScoreQuery and MinScoreQuery nodes on the GPU against the object-level reference (tests/score_nodes_reference.py), bit
for bit: docs, score bits, counts, totalHits and relation.

Generated trees (tests/score_nodes_gen.py) hold both kinds at every depth and under every occur, nested in each other and
at the root, over phrases, numeric and keyword ranges, dismax and msm; MinScoreQuery thresholds are exact scores of
matching docs (or the next float up, NaN, 0). The shard is tests/test_gpu_engines_agree.py's (1.25M docs, window and
slice edges, tf >= 255, positions, keyword columns, deletes) with tests/test_gpu_tree_aggs.py's columns. Every tree entry
point runs: search_tree with and without searchAfter, search_tree_with_collectors (terms with nested min / max / sum and
top hits, min / max / sum, filter collectors) against the aggregation references over the reference's match sets,
score_docs_tree and rescore_query_tree, and a GpuLeafSearcher over three leaves against the whole-shard reference. The
known answers of the reference project's ConstantScoreQueryTest and MinThresholdQueryTest run here too, and refused
calls write no output."""
import math

import numpy as np
import pytest

import oracle
import plan_harness as ph
import query_gen as qg
import rescore_tree_reference as rr
import score_nodes_gen as sg
from helpers import shard_from_token_docs
from nrtsearch_b200 import _native
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, ConstantScoreQuery, GpuIndex, GpuIndexSearcher, GpuLeafSearcher,
                                   MinScoreQuery, Occur, RelevanceCollector, TermQuery, compile_tree)
from score_nodes_reference import ScoreNodeReference
from test_gpu_engines_agree import Truth, build_shard, check
from test_gpu_tree_aggs import Ref, add_columns, check_all, collectors

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
SEEDS = (31, 32, 33)
NQ = 40
N_DOCS = 1_250_000


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    sh = add_columns(build_shard())
    g = GpuIndex(gpu_ctx, sh)
    plane, _ = ph.index_rules(sh.n_docs, sh.term_off)
    df = np.diff(sh.term_off)
    f0 = np.nonzero((sh.term_field == 0) & (df > 0))[0]
    by_df = f0[np.argsort(-df[f0], kind="stable")]
    space = qg.space_of(sh, [(0, False), (3, True)], plane_terms=np.nonzero(plane >= 0)[0][:64], phrase_terms=by_df[20:80])
    yield sh, g, space, ScoreNodeReference(sh), oracle.OracleIndex(sh)
    g.close()


class Matches(Ref):
    """what check_all reads (test_gpu_tree_aggs.Ref), from the object-level reference: every query's live match set and
    scores"""

    def __init__(self, sh, oix, ref, queries):
        self.sh, self.oix = sh, oix
        ev = [ref.eval(q) for q in queries]
        self.present = np.stack([p & ref.live for p, _ in ev])
        self.score = np.stack([s for _, s in ev])
        self._masks = {}


@pytest.fixture(scope="module", params=SEEDS)
def batch(request, corpus):
    sh, g, space, ref, _ = corpus
    seed = request.param
    queries = sg.ScoreNodeGenerator(space, seed, sg.threshold_from(ref)).queries(NQ)
    rng = np.random.default_rng(seed)
    return seed, queries, [Truth(ref, q, rng, sh) for q in queries]


def test_batches_hold_both_kinds(batch):
    seed, queries, truths = batch
    nodes = [w for q in queries for w in sg.wrappers(q)]
    assert sum(isinstance(w, ConstantScoreQuery) for w in nodes) >= 8 and sum(isinstance(w, MinScoreQuery) for w in nodes) >= 8
    totals = np.array([t.total for t in truths])
    assert (totals > 0).mean() > 0.3 and (totals > 1024).any(), f"seed {seed}: {totals}"


@pytest.mark.parametrize("thr", [INT_MAX, 1000])
def test_search_tree(corpus, batch, thr):
    g = corpus[1]
    seed, queries, truths = batch
    s = GpuIndexSearcher(g)
    for k in (1, 7, 100, 1024):
        check(s.search_tree(queries, RelevanceCollector(k, thr)), truths, queries, range(len(queries)), k, thr, seed, "tree")


def test_search_after(corpus, batch):
    g = corpus[1]
    seed, queries, truths = batch
    s = GpuIndexSearcher(g)
    rows = [i for i, t in enumerate(truths) if t.after]
    for v in range(3):   # the page's own key, nextafter up, nextafter down
        res = s.search_tree([queries[i] for i in rows], RelevanceCollector(100, INT_MAX),
                            search_after=[truths[i].after[v][0] for i in rows])
        for row, i in enumerate(rows):
            sd, d, sc, total = truths[i].after[v]
            msg = f"after {sd}: {qg.describe(seed, i, queries[i])}"
            assert int(res.counts[row]) == len(d) and np.array_equal(res.docs[row, :len(d)], d), msg
            assert np.array_equal(res.scores[row, :len(d)].view(np.uint32), sc.view(np.uint32)), msg
            assert int(res.total_hits[row]) == total and res.relation[row] == 0, msg


def test_collectors(corpus, batch):
    sh, g, _, ref, oix = corpus
    seed, queries, truths = batch
    colls = collectors()
    for k in (10, 1024):
        res, outs = GpuIndexSearcher(g).search_tree_with_collectors(queries, RelevanceCollector(k, INT_MAX), colls)
        check(res, truths, queries, range(len(queries)), k, INT_MAX, seed, "tree collectors")
    check_all(Matches(sh, oix, ref, queries), res, outs, colls, 1024, f"seed {seed}")


def test_second_pass(corpus, batch):
    g, ref = corpus[1], corpus[3]
    seed, queries, truths = batch
    s = GpuIndexSearcher(g)
    hits = np.stack([t.hits for t in truths]).astype(np.int32)
    m, sc = s.score_docs_tree(queries, hits)
    for i, t in enumerate(truths):
        msg = f"score_docs_tree: {qg.describe(seed, i, queries[i])}"
        assert np.array_equal(m[i] != 0, t.hit_match), f"{msg}: match flags differ"
        assert np.array_equal(sc[i].view(np.uint32), t.hit_score.view(np.uint32)), f"{msg}: scores differ"
    # rescore each query's reference page (top 100) with the next query of the batch
    n = 100
    docs = np.zeros((len(truths), n), np.int32)
    first = np.zeros((len(truths), n), np.float32)
    counts = np.array([min(len(t.docs), n) for t in truths], np.int32)
    for i, t in enumerate(truths):
        docs[i, :counts[i]], first[i, :counts[i]] = t.docs[:counts[i]], t.scores[:counts[i]]
    rescore = queries[1:] + queries[:1]
    wm, ws = np.zeros(docs.shape, np.uint8), np.zeros(docs.shape, np.float32)
    for i, q in enumerate(rescore):
        p, s_ = ref.eval(q)
        live = p & ref.live
        wm[i], ws[i] = live[docs[i]], np.where(live[docs[i]], s_[docs[i]], np.float32(0))
    for window in (1, 40, 100):
        d, sc, c = s.rescore_query_tree(rescore, docs, first, counts, window, 1.0, 2.0)
        wd, wsc, wc = rr.rescore(docs, first, wm, ws, counts, window, 1.0, 2.0)
        assert np.array_equal(c, wc), f"seed {seed} window {window}: counts"
        for q in range(len(truths)):
            k = int(wc[q])
            msg = f"rescore window {window}: {qg.describe(seed, q, rescore[q])}"
            assert np.array_equal(d[q, :k], wd[q, :k]) and np.array_equal(sc[q, :k].view(np.uint32), wsc[q, :k].view(np.uint32)), msg


def test_leaf_searcher(gpu_ctx, corpus, batch):
    sh, _, _, ref, oix = corpus
    seed, queries, truths = batch
    cuts = [0, 400_000 + 5_000, 1_048_576 + 3, N_DOCS]   # 405,000 is inside a 16,384-doc window
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    try:
        ls = GpuLeafSearcher(gpu_ctx, leaves)
        for k in (7, 100):
            check(ls.search_tree(queries, RelevanceCollector(k, INT_MAX)), truths, queries, range(len(queries)), k, INT_MAX,
                  seed, "3 leaves, tree")
        colls = collectors()
        res, outs = ls.search_tree_with_collectors(queries, RelevanceCollector(10, INT_MAX), colls)
        check(res, truths, queries, range(len(queries)), 10, INT_MAX, seed, "3 leaves, tree collectors")
        check_all(Matches(sh, oix, ref, queries), res, outs, colls, 10, f"3 leaves seed {seed}")
        ls.close()
    finally:
        for x in leaves:
            x.close()


# ---------------------------------------------------------------- known answers and refusals

def test_known_answers(gpu_ctx):
    sh, v = shard_from_token_docs([[d.split() for d in ("t1 t2 t3", "t1 t3", "t4 t5 t6", "t2 t6 t7", "t1 t2 t8")]])
    g = GpuIndex(gpu_ctx, sh)
    try:
        res = GpuIndexSearcher(g).search_tree([ConstantScoreQuery(TermQuery(v[(0, "t2")])),
                                               BoostQuery(ConstantScoreQuery(TermQuery(v[(0, "t2")])), 5.0)],
                                              RelevanceCollector(10, INT_MAX))
        assert res.counts.tolist() == [3, 3] and res.docs[:, :3].tolist() == [[0, 3, 4]] * 2
        assert res.scores[0, :3].tolist() == [1.0] * 3 and res.scores[1, :3].tolist() == [5.0] * 3
    finally:
        g.close()
    sh, v = shard_from_token_docs([[d.split() for d in ("test document one", "test test document two",
                                                          "test test test document three")]])
    g = GpuIndex(gpu_ctx, sh)
    try:
        test = TermQuery(v[(0, "test")])
        s = GpuIndexSearcher(g)
        plain = s.search_tree([test], RelevanceCollector(10, INT_MAX))
        res = s.search_tree([MinScoreQuery(test, 0.5), MinScoreQuery(test, 0.0)], RelevanceCollector(10, INT_MAX))
        n0 = int(plain.counts[0])
        assert n0 == 3 and set(res.docs[0, :res.counts[0]].tolist()) <= set(plain.docs[0, :n0].tolist())
        assert (res.scores[0, :res.counts[0]] >= np.float32(0.5)).all()
        assert res.docs[1, :n0].tolist() == plain.docs[0, :n0].tolist()
        assert np.array_equal(res.scores[1, :n0].view(np.uint32), plain.scores[0, :n0].view(np.uint32))
        want = ScoreNodeReference(sh).search([MinScoreQuery(test, 0.5)], 10)
        assert res.counts[0] == want[2][0] and np.array_equal(res.scores[0].view(np.uint32), want[1][0].view(np.uint32))
    finally:
        g.close()


def test_refused_calls_write_nothing(corpus):
    g = corpus[1]
    s = GpuIndexSearcher(g)
    for call in (lambda q: s.search_tree(q, RelevanceCollector(10, INT_MAX)), lambda q: s.score_docs_tree(q, np.zeros((1, 4), np.int32))):
        with pytest.raises(ValueError, match="MinScoreQuery.min_score must be a non-negative number"):
            call([BooleanQuery().add(MinScoreQuery(TermQuery(1), -1.0), Occur.SHOULD)])
        with pytest.raises(ValueError, match="Boost must be a finite number"):
            call([BoostQuery(ConstantScoreQuery(TermQuery(1)), math.inf)])
    lib = _native.gpu_lib()
    for field, value, msg in (("min_score", -1.0, "MinScoreQuery.min_score"), ("boost", math.nan, "Boost must be a finite number"),
                              ("kind", 5, "bad node kind")):
        carr, ncl, narr, nn, qarr, nq = compile_tree([BooleanQuery().add(MinScoreQuery(TermQuery(1), 1.0), Occur.SHOULD)])
        setattr(narr[0], field, value)
        out = [np.full(10, 77, np.int32), np.full(10, 7.5, np.float32), np.full(1, 77, np.int32), np.full(1, 77, np.int64),
               np.full(1, 77, np.uint8), np.full(1, 77, np.uint8), np.full(1, 77, np.uint8)]
        rc = lib.nrtgpu_search_tree(g.handle, carr, ncl, narr, nn, qarr, nq, 10, INT_MAX, 0, None, None, *[o.ctypes.data for o in out])
        assert rc == 1 and msg in lib.nrtgpu_last_error().decode()
        for o, x in zip(out, (77, 7.5, 77, 77, 77, 77, 77)):
            assert (o == x).all(), "a refused call wrote output"
