"""Sorted top hits (TopHitsCollector with a querySort; nrtgpu_search_bool_aggs_sorted_hits and the searcher's) against
tests/sorted_hits_reference.py over the oracle's match sets and scores.

The shard is the sorted-search shard of tests/sort_single_shard.py (8 % deletes, missing values, a multi-valued column, a
3,000-doc tie group on every sortable column) with a 13-value bucket column added, searched as one image and as the uneven
leaves of tests/searcher_leaves.py (a cut inside the tie group, a leaf of 37 docs). Collectors sit under terms buckets,
under filters and filters in filters, and at the top level, with one-field and multi-field Sorts, a multi-valued column,
missing values, a leading score with and without reverse, and start_hit > 0. Docs, FieldDoc values, counts and totals are
exact, scores NaN; a leading score's value is the float the top-level hit list gives the doc. Relevance top hits in the
same call equal nrtgpu_search_bool_aggs_filtered's bit for bit. Refused calls write nothing."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import filter_aggs_reference as far
import nested_aggs_reference as nr
import oracle
import searcher_leaves as sl
import sort_single_shard as ss
import sorted_hits_reference as ref
from nrtsearch_b200 import NrtGpuError
from nrtsearch_b200 import _native
from nrtsearch_b200.search import (FilterCollector, GpuIndex, GpuIndexSearcher, GpuLeafSearcher, MatchAllDocsQuery, RangeQuery,
                                   RelevanceCollector, SortType, TermsCollector, TopHitsCollector, ValueSetFilter, MinCollector,
                                   _FilteredRecords, compile_queries)

pytestmark = pytest.mark.gpu
INVALID = 1
INT_MAX = 2**31 - 1
K = 10
BKT = 10   # the added bucket column: 13 values
SORTS = {
    "i32": [SortType(ss.C_I32, field_type="int")],
    "mv-max-desc": sl.multi_sorts()["mv-max-desc"],
    "score": sl.multi_sorts()["score"],
    "score-reverse,i32": sl.multi_sorts()["score-reverse,i32"],
    "score,mv-max,i64": sl.multi_sorts()["score,mv-max,i64"],
    "f64,docid-desc,i64": sl.multi_sorts()["f64,docid-desc,i64"],
    "8 fields": sl.multi_sorts()["8 fields"],
}
FILTER_Q = RangeQuery(ss.C_I32, -1000, 3000)
FILTER_SET = ValueSetFilter(BKT, (1, 2, 3, 4, 5, 6))


@pytest.fixture(scope="module")
def setup(gpu_ctx):
    sh = ss.make_shard(sl.N, sl.DOC_BASE, sl.TIE_LO)
    sh.columns = list(sh.columns) + [np.arange(sh.n_docs, dtype=np.int64) * 7919 % 13]
    sh.column_has = list(sh.column_has) + [None]
    sh.column_offsets = list(sh.column_offsets) + [None]
    whole = GpuIndex(gpu_ctx, sh)
    cuts = sl.cuts()
    leaves = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    s = GpuLeafSearcher(gpu_ctx, leaves)
    yield sh, oracle.OracleIndex(sh), whole, leaves, s
    s.close()
    for g in leaves + [whole]:
        g.close()


def searcher(setup, target):
    _, _, whole, _, s = setup
    return GpuIndexSearcher(whole) if target == "whole" else s


class Ref:
    """match sets, oracle scores and filter masks of a batch, computed once per query"""

    def __init__(self, sh, oix, queries):
        self.sh, self.oix = sh, oix
        self.carr, _, self.qarr, self.nq = compile_queries(queries)
        self._m, self._s = {}, {}

    def match(self, q):
        if q not in self._m:
            self._m[q] = oracle.match_bitmap(self.oix, self.carr, self.qarr, q).astype(bool)
        return self._m[q]

    def scores(self, q):
        if q not in self._s:
            self._s[q] = nr.query_scores(self.sh, self.oix, self.carr, self.qarr, q, self.match(q))
        return self._s[q]

    def mask(self, f):
        if isinstance(f, ValueSetFilter):
            return far.value_set_mask(self.sh, f.column, f.sortable()).astype(bool)
        carr, _, qarr, _ = compile_queries([f])
        return far.query_mask(self.oix, carr, qarr, 0).astype(bool)


def check_hits(r, at, R, q, c, bucket, what):
    docs = np.nonzero(bucket)[0]
    fields = None if c.sort is None else sl.ref_fields(c.sort_fields())
    want, vals = ref.top_hits(R.sh, docs, R.scores(q)[docs], fields, c.top_hits, c.start_hit)
    m = len(want)
    assert r["counts"][at] == m and r["total_hits"][at] == len(docs), f"{what}: counts {r['counts'][at]} / {m}"
    assert r["docs"][at][:m].tolist() == want.tolist(), f"{what}: docs"
    assert not r["docs"][at][m:].any(), f"{what}: docs past the count"
    if c.sort is None:
        assert np.array_equal(r["scores"][at][:m].view(np.uint32), R.scores(q)[want - R.sh.doc_base].view(np.uint32)), what
        assert "sort_values" not in r
    else:
        assert np.isnan(r["scores"][at]).all(), f"{what}: scores"
        assert np.array_equal(r["sort_values"][at][:m], vals), f"{what}: values"
        assert not r["sort_values"][at][m:].any(), f"{what}: values past the count"


def check(R, q, c, o, bucket, what):
    """collector c's result o for query q over the docs `bucket` its parent hands it"""
    if isinstance(c, TopHitsCollector):
        check_hits(o, q, R, q, c, bucket, what)
    elif isinstance(c, FilterCollector):
        b = bucket & R.mask(c.filter)
        assert o["doc_count"][q] == b.sum(), what
        for name, x in c.nested:
            check(R, q, x, o[name], b, f"{what}/{name}")
    else:
        col = np.asarray(R.sh.columns[c.column])
        for i in range(o["n"][q]):
            b = bucket & (col == o["keys"][q, i])
            assert o["counts"][q, i] == b.sum(), what
            for name, x in c.nested:
                if isinstance(x, TopHitsCollector):
                    check_hits(o["nested"][name], (q, i), R, q, x, b, f"{what}/{name} slot {i}")


def request(sort):
    return [TermsCollector(BKT, 5, nested=(("h", TopHitsCollector(7, 2, sort)), ("r", TopHitsCollector(4)))),
            FilterCollector(FILTER_Q, (("h", TopHitsCollector(6, 0, sort)),
                                       ("f", FilterCollector(FILTER_SET, (("t", TermsCollector(BKT, 3, nested=(
                                           ("h", TopHitsCollector(5, 1, sort)),))),))))),
            TopHitsCollector(10, 3, sort)]


def unsorted(c):
    if isinstance(c, TopHitsCollector):
        return dataclasses.replace(c, sort=None)
    if isinstance(c, (TermsCollector, FilterCollector)):
        return dataclasses.replace(c, nested=tuple((n, unsorted(x)) for n, x in c.nested))
    return c


def run_filtered(setup, target, queries, additional):
    """the same request through nrtgpu_search_bool_aggs_filtered / the searcher's (no sorts)"""
    _, _, whole, _, s = setup
    carr, ncl, qarr, nq = compile_queries(queries)
    fr = _FilteredRecords(nq, additional)
    docs, scores = np.zeros((nq, K), np.int32), np.zeros((nq, K), np.float32)
    counts, total = np.zeros(nq, np.int32), np.zeros(nq, np.int64)
    lib = _native.gpu_lib()
    args = fr.args
    if target == "whole":
        rc = lib.nrtgpu_search_bool_aggs_filtered(whole.handle, carr, ncl, qarr, nq, K, 0, *args, None, docs.ctypes.data,
                                                  scores.ctypes.data, counts.ctypes.data, total.ctypes.data)
    else:
        rc = lib.nrtgpu_searcher_search_bool_aggs_filtered(s.handle, carr, ncl, qarr, nq, K, 0, *args, None, docs.ctypes.data,
                                                           scores.ctypes.data, counts.ctypes.data, total.ctypes.data)
    assert rc == 0, lib.nrtgpu_last_error()
    return docs, scores, counts, total, fr.outs


@pytest.mark.parametrize("target", ["whole", "leaves"])
@pytest.mark.parametrize("sort_id", list(SORTS))
def test_sorted_top_hits(setup, target, sort_id):
    sh, oix, *_ = setup
    queries = ss.QUERIES
    adds = request(SORTS[sort_id])
    res, outs = searcher(setup, target).search_with_collectors(queries, RelevanceCollector(K, INT_MAX), adds)
    R = Ref(sh, oix, queries)
    for q in range(len(queries)):
        m = R.match(q)
        assert res.total_hits[q] == m.sum()
        n = res.counts[q]   # the top-level hit list: its scores are the ones a leading SCORE carries
        assert np.array_equal(res.scores[q, :n].view(np.uint32), R.scores(q)[res.docs[q, :n] - sh.doc_base].view(np.uint32))
        for i, c in enumerate(adds):
            check(R, q, c, outs[i], m, f"{target} {sort_id} q{q} aggs[{i}]")
        assert outs[2]["total_hits"][q] == res.total_hits[q]   # a top-level collector sees every collected doc
    # the relevance results of the call are those of the call without Sorts
    docs, scores, counts, total, plain = run_filtered(setup, target, queries, [unsorted(c) for c in adds])
    assert np.array_equal(docs, res.docs) and np.array_equal(scores.view(np.uint32), res.scores.view(np.uint32))
    assert np.array_equal(counts, res.counts) and np.array_equal(total, res.total_hits)
    for k in ("docs", "scores", "counts", "total_hits"):
        a, b = outs[0]["nested"]["r"][k], plain[0]["nested"]["r"][k]
        assert np.array_equal(a.view(np.uint32) if k == "scores" else a, b.view(np.uint32) if k == "scores" else b), k
    assert np.array_equal(outs[0]["keys"], plain[0]["keys"]) and np.array_equal(outs[1]["doc_count"], plain[1]["doc_count"])


@pytest.mark.parametrize("target", ["whole", "leaves"])
def test_several_pass2_groups(setup, target):
    """about 1.1M keys per match-all query: 170 of them take three groups of the 2^26-key budget"""
    sh, oix, *_ = setup
    queries = [MatchAllDocsQuery()] * 170 + [RangeQuery(ss.C_I32, 17, 18)]
    sort = SORTS["score,mv-max,i64"]
    adds = [TermsCollector(BKT, 13, nested=(("h", TopHitsCollector(3, 1, sort)), ("r", TopHitsCollector(2))))]
    res, outs = searcher(setup, target).search_with_collectors(queries, RelevanceCollector(K, INT_MAX), adds)
    R = Ref(sh, oix, queries)
    for q in (0, 85, 169, 170):
        check(R, q, adds[0], outs[0], R.match(q), f"{target} q{q}")


def raw_call(setup, target, queries, additional, mutate):
    """a direct call with sentinel-filled outputs after mutate(records); returns (status, message, whether any output changed)"""
    sh, _, whole, leaves, s = setup
    carr, ncl, qarr, nq = compile_queries(queries)
    idx = whole if target == "whole" else None
    orders_of = (lambda f: (C.c_void_p * 1)(whole.sort_order(f).value)) if target == "whole" else \
        (lambda f: (C.c_void_p * len(leaves))(*[l.sort_order(f).value for l in leaves]))
    fr = _FilteredRecords(nq, additional, orders_of)
    args = list(fr.sorted_args)
    mutate(fr, args)
    outs = [np.full((nq, K), -7, np.int32), np.full((nq, K), -7.0, np.float32), np.full(nq, -7, np.int32), np.full(nq, -7, np.int64)]
    bufs = []

    def collect(o):
        if isinstance(o, dict):
            for v in o.values():
                collect(v)
        else:
            o.fill(-7)
            bufs.append(o)
    for o in fr.outs:
        collect(o)
    lib = _native.gpu_lib()
    fn = lib.nrtgpu_search_bool_aggs_sorted_hits if idx is not None else lib.nrtgpu_searcher_search_bool_aggs_sorted_hits
    rc = fn(idx.handle if idx is not None else s.handle, carr, ncl, qarr, nq, K, 0, *args, None, *[o.ctypes.data for o in outs])
    msg = lib.nrtgpu_last_error().decode() if rc else ""
    changed = any((o != -7).any() for o in outs + bufs)
    return rc, msg, changed


def test_refusals_write_nothing(setup):
    sh, _, whole, leaves, s = setup
    queries = ss.QUERIES[:3]
    sort = SORTS["i32"]
    adds = [TermsCollector(BKT, 4, nested=(("h", TopHitsCollector(3, 0, sort)), ("m", MinCollector(ss.C_I32, "int"))))]

    def order_on_min(fr, args):
        args[6][1].orders = args[6][0].orders
    for target in ("whole", "leaves"):
        rc, msg, changed = raw_call(setup, target, queries, adds, order_on_min)
        assert rc == INVALID and "only top hits take a sort order" in msg and not changed, (target, msg)
    # an order made on another index (a leaf's order on the whole image)

    def leaf_order(fr, args):
        fr.keep.append((C.c_void_p * 1)(leaves[0].sort_order(sort).value))
        args[6][0].orders = C.cast(fr.keep[-1], C.c_void_p)
    rc, msg, changed = raw_call(setup, "whole", queries, adds, leaf_order)
    assert rc == INVALID and "another index" in msg and not changed, msg
    # leaves: orders swapped between two leaves, of different Sorts, a NULL order

    def swapped(fr, args):
        arr = (C.c_void_p * len(leaves))(*[l.sort_order(sort).value for l in leaves])
        arr[0], arr[1] = arr[1], arr[0]
        fr.keep.append(arr)
        args[6][0].orders = C.cast(arr, C.c_void_p)

    def mixed(fr, args):
        arr = (C.c_void_p * len(leaves))(*[l.sort_order(sort if i else SORTS["8 fields"]).value for i, l in enumerate(leaves)])
        fr.keep.append(arr)
        args[6][0].orders = C.cast(arr, C.c_void_p)

    def null(fr, args):
        arr = (C.c_void_p * len(leaves))(*[l.sort_order(sort).value for l in leaves])
        arr[2] = None
        fr.keep.append(arr)
        args[6][0].orders = C.cast(arr, C.c_void_p)
    for mutate, text in ((swapped, "leaf 0 was made on another index"), (mixed, "different Sorts"), (null, "NULL sort order")):
        rc, msg, changed = raw_call(setup, "leaves", queries, adds, mutate)
        assert rc == INVALID and text in msg and not changed, msg
    # orders_parent on a sorted top hits keeps the existing refusal
    ordered = [TermsCollector(BKT, 4, nested=(("h", TopHitsCollector(3, 0, sort)),), order_by="h")]
    for target in ("whole", "leaves"):
        rc, msg, changed = raw_call(setup, target, queries, ordered, lambda fr, args: None)
        assert rc == INVALID and "top hits cannot order the buckets" in msg and not changed, msg
        with pytest.raises(NrtGpuError):
            searcher(setup, target).search_with_collectors(queries, RelevanceCollector(K, INT_MAX), ordered)
