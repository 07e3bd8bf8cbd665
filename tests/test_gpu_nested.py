"""NestedQuery (block joins) on the GPU against the object-level reference (tests/nested_reference.py), bit for bit: docs,
score bits, counts and totalHits.

The corpus is a synthetic nested index of about 1.2M docs (two 1M-doc slices of the window engine): blocks of a Poisson
number of children and their parent, two child paths, children after the last parent and parents that also hold a
child path (both join nothing), deletes among children and parents. Generated trees put joins at several depths, under
every occur and inside DISMAX, CONSTANT and MIN_SCORE nodes, in all five score modes, with boosts around them and child
queries holding terms, bools, phrases and ranges. Every accepted tree entry point runs: search_tree (a 1024-query batch
included), prepared batches with set_live_docs between prepare and run and repeated runs, search_tree_with_collectors,
and a GpuLeafSearcher over three leaves cut at block boundaries against the whole-shard reference. Refused calls write
nothing."""
import os
import subprocess
import sys

import numpy as np
import pytest

import nested_reference as nr
from nrtsearch_b200 import NrtGpuError, _native
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, ConstantScoreQuery, DisjunctionMaxQuery, GpuIndex, GpuIndexSearcher,
                                   GpuLeafSearcher, MinScoreQuery, NestedQuery, Occur, PhraseQuery, RangeQuery,
                                   RelevanceCollector, TermQuery, compile_tree)
from test_gpu_score_nodes import Matches
from test_gpu_tree_aggs import add_columns, check_all, collectors

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
S, M, F, N = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
MODES = ("none", "sum", "avg", "max", "min")
N_PARENTS = 280_000
VOCAB = 400


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(c, o)
    return q


class NestedGen:
    """seeded query trees with joins: terms of the Zipf-like vocabulary (common and rare), phrases of two terms, ranges"""

    def __init__(self, paths, seed, common=0.4, rare_from=12):
        self.paths, self.rng, self.common, self.rare_from = paths, np.random.default_rng(seed), common, rare_from

    def term(self):
        r = self.rng
        return TermQuery(int(r.integers(0, 12) if r.random() < self.common else r.integers(self.rare_from, VOCAB)))

    def child(self):
        r = self.rng
        k = r.integers(0, 5)
        if k == 0:
            q = self.term()
        elif k == 1:
            q = bq(*[(self.term(), r.choice([S, S, M])) for _ in range(int(r.integers(2, 4)))])
        elif k == 2:
            a = int(r.integers(0, 30))   # (two different terms: a sloppy phrase with a repeated term is refused)
            q = bq((PhraseQuery([a, (a + 1 + int(r.integers(0, 29))) % 30], slop=int(r.integers(0, 3))), S), (self.term(), S))
        elif k == 3:
            lo = int(r.integers(0, 900_000))
            q = bq((self.term(), M), (RangeQuery(0, lo, lo + int(r.integers(10_000, 400_000))), r.choice([F, S])))
        else:
            q = bq((self.term(), S), (self.term(), S), (self.term(), N))
        if r.random() < 0.3:
            q = BoostQuery(q, float(r.choice([0.5, 2.0, 3.25])))
        return q

    def nested(self):
        r = self.rng
        q = NestedQuery(self.child(), self.paths[int(r.random() < 0.25)], str(r.choice(MODES)))
        return BoostQuery(q, float(r.choice([0.75, 1.5]))) if r.random() < 0.3 else q

    def query(self):
        r = self.rng
        k = r.integers(0, 7)
        if k == 0:
            return self.nested()
        if k == 1:
            return bq((self.term(), M), (self.nested(), S))
        if k == 2:
            return bq((self.nested(), M), (self.term(), S), (self.nested(), r.choice([S, F, N])))
        if k == 3:
            return bq((DisjunctionMaxQuery([self.nested(), self.term()], 0.3), M))
        if k == 4:
            return bq((ConstantScoreQuery(self.nested()), S), (self.term(), S))
        if k == 5:
            return bq((MinScoreQuery(self.nested(), float(r.choice([0.5, 2.0]))), S), (self.term(), S))
        return bq((bq((self.nested(), F), (self.term(), S)), M), (self.term(), S))

    def queries(self, n):
        return [self.query() for _ in range(n)]


@pytest.fixture(scope="module")
def corpus(gpu_ctx):
    sh, paths = nr.build_nested_shard(N_PARENTS, 0x5E5)
    sh = add_columns(sh)
    rng = np.random.default_rng(7)
    sh.live_docs = (rng.random(sh.n_docs) >= 0.05).astype(np.uint8)
    g = GpuIndex(gpu_ctx, sh)
    yield sh, paths, g, nr.NestedReference(sh)
    g.close()


def same(res, want, what):
    d, s, c, t = want
    assert np.array_equal(res.counts, c), f"{what}: counts"
    assert np.array_equal(res.total_hits, t), f"{what}: totalHits"
    for q in range(len(c)):
        n = c[q]
        assert np.array_equal(res.docs[q, :n], d[q, :n]), f"{what} query {q}: docs"
        assert np.array_equal(res.scores[q, :n].view(np.uint32), s[q, :n].view(np.uint32)), f"{what} query {q}: scores"


def test_corpus_spans_two_slices(corpus):
    sh = corpus[0]
    assert sh.n_docs > (1 << 20)
    assert nr.parent_mask(sh).sum() == N_PARENTS


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_generated_trees(corpus, seed):
    sh, paths, g, ref = corpus
    queries = NestedGen(paths, seed).queries(48)
    d, s, c, t = ref.search(queries, 100)
    for k in (10, 100):   # (a page of 10 is the first 10 of the page of 100)
        res = GpuIndexSearcher(g).search_tree(queries, RelevanceCollector(k, INT_MAX))
        same(res, (d[:, :k], s[:, :k], np.minimum(c, k), t), f"seed {seed} k {k}")


def test_batch_of_1024(corpus):
    sh, paths, g, ref = corpus
    # (selective child terms: joins over every child of a path bound 2^26 child matches in a few hundred queries)
    queries = NestedGen(paths, 99, common=0.0, rare_from=40).queries(1024)
    res = GpuIndexSearcher(g).search_tree(queries, RelevanceCollector(10, INT_MAX))
    same(res, ref.search(queries, 10), "1024 queries")


def test_compiled_reference_agrees(corpus):
    """the array-level reference over compile_tree's output and the object-level one give the same pages"""
    sh, paths, g, ref = corpus
    queries = NestedGen(paths, 5).queries(16)
    d, s, c, t, _ = nr.search(sh, queries, 10)
    same(GpuIndexSearcher(g).search_tree(queries, RelevanceCollector(10, INT_MAX)), (d, s, c, t), "compiled reference")


def test_collectors(corpus):
    sh, paths, g, ref = corpus
    queries = NestedGen(paths, 11).queries(24)
    colls = collectors()
    res, outs = GpuIndexSearcher(g).search_tree_with_collectors(queries, RelevanceCollector(10, INT_MAX), colls)
    import oracle
    check_all(Matches(sh, oracle.OracleIndex(sh), ref, queries), res, outs, colls, 10, "collectors")


def test_prepared_live_docs_and_repeats(gpu_ctx, corpus):
    sh, paths, _, _ = corpus
    sh2, _ = nr.build_nested_shard(20_000, 0x77)
    g = GpuIndex(gpu_ctx, sh2)
    try:
        queries = NestedGen(paths, 21).queries(32)
        s = GpuIndexSearcher(g)
        pb = s.prepare_tree(queries, RelevanceCollector(10, INT_MAX))
        try:
            pb.run()
            same(pb.fetch(), nr.NestedReference(sh2).search(queries, 10), "prepared")
            live = (np.random.default_rng(3).random(sh2.n_docs) >= 0.2).astype(np.uint8)
            g.set_live_docs(live)
            sh2.live_docs = live
            want = nr.NestedReference(sh2).search(queries, 10)
            for i in range(3):
                pb.run()
                same(pb.fetch(), want, f"prepared after set_live_docs, run {i}")
            for i in range(2):
                same(s.search_tree(queries, RelevanceCollector(10, INT_MAX)), want, f"one-shot run {i}")
        finally:
            pb.close()
    finally:
        g.close()


def test_leaf_searcher(gpu_ctx, corpus):
    sh, paths, _, ref = corpus
    cuts = nr.block_cuts(sh, 3, np.random.default_rng(4))
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    try:
        ls = GpuLeafSearcher(gpu_ctx, leaves)
        queries = NestedGen(paths, 31).queries(32)
        same(ls.search_tree(queries, RelevanceCollector(10, INT_MAX)), ref.search(queries, 10), "3 leaves")
        colls = collectors()
        res, outs = ls.search_tree_with_collectors(queries, RelevanceCollector(10, INT_MAX), colls)
        import oracle
        check_all(Matches(sh, oracle.OracleIndex(sh), ref, queries), res, outs, colls, 10, "3 leaves collectors")
        ls.close()
    finally:
        for l in leaves:
            l.close()


def _raw_call(g, q, mutate=None):
    """nrtgpu_search_tree on compile_tree's arrays (mutated first), into outputs filled with 77: (rc, outputs)"""
    lib = _native.gpu_lib()
    carr, ncl, narr, nn, qarr, nq = compile_tree([q])
    if mutate:
        mutate(carr, narr)
    out = [np.full(10, 77, np.int32), np.full(10, 7.5, np.float32), np.full(1, 77, np.int32), np.full(1, 77, np.int64),
           np.full(1, 77, np.uint8), np.full(1, 77, np.uint8), np.full(1, 77, np.uint8)]
    rc = lib.nrtgpu_search_tree(g.handle, carr, ncl, narr, nn, qarr, nq, 10, INT_MAX, 0, None, None, *[o.ctypes.data for o in out])
    return rc, lib.nrtgpu_last_error().decode(), out


def _untouched(out):
    for o, x in zip(out, (77, 7.5, 77, 77, 77, 77, 77)):
        assert (o == x).all(), "a refused call wrote output"


def test_refused_calls_write_nothing(gpu_ctx, corpus):
    sh, paths, g, _ = corpus
    nq_ = NestedQuery(TermQuery(3), paths[0], "sum")

    def set_mode(m):
        def f(carr, narr):
            narr[0].min_should_match = m
        return f

    def second_clause(carr, narr):
        narr[0].clause_end = narr[0].clause_begin + 2

    def must_not(carr, narr):
        carr[narr[0].clause_begin].occur = int(N)

    for mutate, code, msg in ((set_mode(5), 1, "score mode"), (set_mode(-1), 1, "score mode"),
                              (second_clause, 1, "exactly one clause"), (must_not, 1, "must be MUST")):
        rc, err, out = _raw_call(g, bq((nq_, M)), mutate)
        assert rc == code and msg in err, (rc, err)
        _untouched(out)
    # a join inside a join's child query
    rc, err, out = _raw_call(g, bq((NestedQuery(bq((nq_, M)), paths[0], "max"), M)))
    assert rc == 3 and "inside a NestedQuery" in err
    _untouched(out)
    # an image without parents
    sh2, _ = nr.build_nested_shard(50, 9)
    sh2.parent_term = None
    g2 = GpuIndex(gpu_ctx, sh2)
    try:
        rc, err, out = _raw_call(g2, bq((nq_, M)))
        assert rc == 1 and "index has no parent docs" in err
        _untouched(out)
    finally:
        g2.close()
    # tree rescoring answers "bad node kind"
    with pytest.raises(NrtGpuError, match="bad node kind"):
        GpuIndexSearcher(g).score_docs_tree([bq((nq_, M))], np.zeros((1, 4), np.int32))


_CAP_SCRIPT = """
import sys
sys.path[:0] = sys.argv[1:3]
import numpy as np
import nested_reference as nr
from nrtsearch_b200 import NrtGpuUnsupported
from nrtsearch_b200.search import GpuContext, GpuIndex, GpuIndexSearcher, NestedQuery, RelevanceCollector, TermQuery
sh, paths = nr.build_nested_shard(2000, 5)
ctx = GpuContext(0)
g = GpuIndex(ctx, sh)
s = GpuIndexSearcher(g)
small = [NestedQuery(TermQuery(350), paths[0], "sum")]
s.search_tree(small, RelevanceCollector(10, 2**31 - 1))
try:
    s.search_tree([NestedQuery(TermQuery(0), paths[0], "sum")], RelevanceCollector(10, 2**31 - 1))
    print("ACCEPTED")
except NrtGpuUnsupported as e:
    print("REFUSED", "child matches, more than 50" in str(e))
g.close()
ctx.close()
"""


def test_env_lowers_the_join_cap():
    """NRTGPU_JOIN_CHILDREN, read when the context is created, lowers the per-call cap of bounded child matches"""
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, NRTGPU_JOIN_CHILDREN="50")
    out = subprocess.run([sys.executable, "-c", _CAP_SCRIPT, here, os.path.dirname(here)], env=env, capture_output=True,
                         text=True, timeout=600)
    assert out.returncode == 0, out.stderr
    assert out.stdout.split()[-2:] == ["REFUSED", "True"], out.stdout
