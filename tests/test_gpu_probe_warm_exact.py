"""Exact sweep warm-ups of posting_probe_kernel (TOP_SCORES pure disjunctions whose lists other than the rarest all
have tf planes): the warm-up scores, counts and outputs the docs of the rarest list up to the first granule boundary
with 32K of its postings below it, and the query's other items skip them. The shard has a rarest list shorter than 32K
postings (the warm-up covers the whole shard) and one of 60K spread over the shard (the warm-up ends inside slice 1,
inside a part of the split (query, slice) pairs), with dense lists beside them; the batch also holds a query with a
list without a plane and a query of one list (lower-bound warm-ups) and a conjunction. Pages are compared with the
exhaustive oracle, with a threshold that prunes and one that never does (every list leads: ownership of the prefix docs
by the warm-up, exact totals), without and with deletes; the profiling counters show the exact warm-ups ran."""
import dataclasses
import re

import numpy as np
import pytest

import plan_harness as ph
import probe_edge_shards as pe
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import GpuIndex, GpuIndexSearcher, Occur, RelevanceCollector
from test_batch_plan import shard_dictionary
from test_gpu_probe_edges import THR, _context, check, same, want_pages
from test_plan_warm_exact import warm_plan

pytestmark = pytest.mark.gpu
N_DOCS = 1_500_007          # 3 slices; tf planes from N_DOCS / 64 = 23,438 postings
NO_PRUNE = 1_000_000_000    # TOP_SCORES, but more than any query's hits: MAXSCORE never starts, totals are exact
REP = 8                     # more work items than resident CTAs
_EXACT = re.compile(r"\[nrtgpu probe simple\] exact warm-ups: (\d+) items, (\d+) driver postings")


def warm_shard():
    rng = np.random.default_rng(23)
    im = pe._Image()
    lists = {}
    for name, df in (("W_SHORT", 9_000), ("W_LONG", 60_000), ("NOPLANE", 15_000), ("P1", 150_000), ("P2", 420_000)):
        d = np.sort(rng.choice(N_DOCS, df, replace=False))
        lists[name] = d
        im.add(name, d, pe._tf_cycle(d, df))
    lens = rng.integers(3, 40, N_DOCS)
    return im.shard(N_DOCS, [ix.TextField(pe._BYTE4[lens], N_DOCS, int(lens.sum()))]), lists


@pytest.fixture(scope="module")
def warm():
    return warm_shard()


def queries(b):
    t = b.term
    return [pe.disj(t["W_SHORT"], t["P1"], t["P2"]),                   # exact: the warm-up covers the whole shard
            pe.disj(t["W_LONG"], t["P1"], t["P2"]),                    # exact: it ends inside slice 1
            pe.disj(t["P2"], t["W_LONG"]),                             # exact, the warm-up's list in slot 1
            pe.disj(t["W_LONG"]),                                      # one list: a lower-bound warm-up
            pe.disj(t["W_SHORT"], t["NOPLANE"], t["P1"]),              # NOPLANE has no plane: a lower-bound warm-up
            pe.bq((t["W_LONG"], Occur.MUST), (t["P1"], Occur.MUST))]   # generic
N_EXACT = 3


def warm_gran(lists):
    """end granule of W_LONG's exact warm-up: the first granule boundary with 32,768 of its postings below it"""
    return (int(lists["W_LONG"][32_767]) >> 10) + 1


def test_exact_warm_up_ends_inside_a_split_slice(warm):
    """The premise of the shard: the (query, slice) pairs are split into parts, and W_LONG's warm-up ends strictly
    inside a part of slice 1, so an item of its query straddles the end."""
    b, lists = warm
    assert len(lists["W_SHORT"]) < 32_768
    qs = queries(b)
    g_w = warm_gran(lists)
    straddle = []
    with warm_plan(shard_dictionary(b.shard), qs, 40, THR) as (p, exact):
        assert exact.tolist() == [0, 0, 1, -1, -1, -1]
        gps = p.slice_docs // 1024
        for q, w in zip(p.work_query, p.work_item):
            sl, _, lparts, flags, _ = ph.decode(w)
            g_lo, g_hi = p.span(w)[:2]
            if q == 1 and not flags and g_lo < g_w - sl * gps < g_hi:
                straddle.append((sl, lparts))
    assert len(straddle) == 1 and straddle[0][0] == 1 and straddle[0][1] > 0, straddle


@pytest.mark.parametrize("deletes", [False, True], ids=["live", "deletes"])
@pytest.mark.parametrize("threshold", [THR, NO_PRUNE], ids=["pruned", "no_prune"])
@pytest.mark.parametrize("top_k", [1, 40, 512])
def test_exact_warm_ups_match_oracle(gpu_ctx, warm, capfd, top_k, threshold, deletes):
    b, lists = warm
    base = queries(b)
    qs = list(base) * REP
    live = None
    shard = b.shard
    if deletes:
        live = np.ones(N_DOCS, np.uint8)
        live[::5] = 0
        shard = dataclasses.replace(b.shard, live_docs=live)
    want = tuple(np.concatenate([a] * REP) for a in want_pages(b, "warm", base, top_k, live=live))
    dbg = _context(NRTGPU_DEBUG_MODES="1")
    res = {}
    try:
        for name, ctx in (("auto", gpu_ctx), ("dbg", dbg)):
            gix = GpuIndex(ctx, shard)
            try:
                capfd.readouterr()
                res[name] = GpuIndexSearcher(gix).search_batch(qs, RelevanceCollector(top_k, threshold))
                err = capfd.readouterr().err
            finally:
                gix.close()
    finally:
        dbg.close()
    what = f"k={top_k} thr={threshold} deletes={deletes}"
    check(res["auto"], want, threshold, what)
    same(res["dbg"], res["auto"], f"{what}: profiling instantiation")
    if threshold == NO_PRUNE:
        assert (res["auto"].relation == 0).all(), f"{what}: a query was pruned"
        assert np.array_equal(res["auto"].total_hits, want[3]), f"{what}: totalHits"
    m = _EXACT.search(err)
    assert m and int(m.group(1)) == N_EXACT * REP, f"{what}: exact warm-ups: {err[-800:]}"
    below = int(np.searchsorted(lists["W_LONG"], warm_gran(lists) * 1024))   # W_LONG postings below the end granule
    assert int(m.group(2)) == REP * (len(lists["W_SHORT"]) + 2 * below), f"{what}: exact warm-up postings"
