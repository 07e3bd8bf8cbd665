"""posting_probe_kernel on shards built on its structural edges (tests/probe_edge_shards.py; the plan-side facts are
proved on the CPU by tests/test_probe_edges_plan.py): clustered long lists that force one-granule runs, short lists on
both sides of the stage limits of both launch configurations, lists at every post_base mod 16, the index-build rule
edges, postings at every granule / slice edge and n - 1 on a shard with a partial last granule and plane byte, every tf
class, docs at the shortest field length, a tie group across part and slice edges, an omitNorms field, 16-way split
items behind a warm-up item with searchAfter. Every page is compared with the exhaustive oracle, in both score modes,
at top_k 1, 40 and 512, through configurations A and B and the automatic choice, through 3 leaves, and through a
PreparedBatch reused across a deletes update. The kernel's own counters (NRTGPU_DEBUG_MODES) prove that the runs,
staging and flushes happened."""
import dataclasses
import os
import re

import numpy as np
import pytest

import oracle
import plan_harness as ph
import probe_edge_shards as pe
from helpers import assert_same_hits
from nrtsearch_b200.search import (GpuContext, GpuIndex, GpuIndexSearcher, GpuLeafSearcher, RelevanceCollector, ScoreDoc,
                                   compile_queries)
from test_batch_plan import shard_dictionary

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
THR = 50                     # TOP_SCORES: pruning as soon as 50 (or top_k) hits are known
TOP_KS = (1, 40, 512)
REP = 8                      # batches run 8 copies of their queries: with more work items than resident CTAs, most items
                             # start after their query's warm-up published a threshold (MAXSCORE roles, tf-pattern bounds)


def rep(qs):
    return list(qs) * REP


def tile(want):
    return tuple(np.concatenate([a] * REP) for a in want)


def _context(**env):
    """GpuContext with NRTGPU_* variables set only while nrtgpu_init reads them."""
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return GpuContext(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def edge():
    return pe.edge_shard()


@pytest.fixture(scope="module")
def contexts(gpu_ctx, edge):
    """default / A / B / debug contexts, each with the edge shard's image"""
    made = {"A": _context(NRTGPU_PROBE_CFG="1"), "B": _context(NRTGPU_PROBE_CFG="2"), "dbg": _context(NRTGPU_DEBUG_MODES="1")}
    ctxs = {"auto": gpu_ctx, **made}
    idx = {k: GpuIndex(c, edge.shard) for k, c in ctxs.items()}
    yield ctxs, idx
    for g in idx.values():
        g.close()
    for c in made.values():
        c.close()


_ORACLE = {}


def want_pages(b, key, qs, k, search_after=None, live=None):
    ck = (id(b), key, k, live is not None)
    if search_after is not None or ck not in _ORACLE:
        sh = b.shard if live is None else dataclasses.replace(b.shard, live_docs=live)
        carr, ncl, qarr, nq = compile_queries(qs, search_after)
        w = oracle.search_compiled(oracle.OracleIndex(sh), carr, ncl, qarr, nq, k)
        if search_after is not None:
            return w
        _ORACLE[ck] = w
    return _ORACLE[ck]


def as_tuple(r):
    return r.docs, r.scores, r.counts, r.total_hits, r.relation


def check(got, want, threshold, what):
    """Same pages as the oracle; EQUAL_TO totals exact, GREATER_THAN_OR_EQUAL_TO above the threshold and <= the exact count."""
    g = as_tuple(got)
    assert_same_hits(g, want, what=what)
    gte = got.relation != 0
    if threshold == INT_MAX:
        assert not gte.any(), f"{what}: COMPLETE reported GREATER_THAN_OR_EQUAL_TO"
    assert (got.total_hits[gte] > threshold).all() and (got.total_hits[gte] <= want[3][gte]).all(), f"{what}: lower bound"


def same(a, b, what):
    """Bit-identical pages; totals equal where both are EQUAL_TO (a pruned count is a lower bound that depends on when
    each work item saw its query's threshold)."""
    assert np.array_equal(a.counts, b.counts), what
    for q in range(len(a.counts)):
        n = int(a.counts[q])
        assert np.array_equal(a.docs[q, :n], b.docs[q, :n]), f"{what} query {q}"
        assert np.array_equal(a.scores[q, :n].view(np.uint32), b.scores[q, :n].view(np.uint32)), f"{what} query {q}"
    eq = (a.relation == 0) & (b.relation == 0)
    assert np.array_equal(a.total_hits[eq], b.total_hits[eq]), what


@pytest.mark.parametrize("threshold", [THR, INT_MAX], ids=["top_scores", "complete"])
@pytest.mark.parametrize("top_k", TOP_KS)
@pytest.mark.parametrize("batch", ["disj", "conj", "dense"])
def test_edge_batches_match_oracle_in_every_configuration(contexts, edge, batch, top_k, threshold):
    """Every batch, page-for-page equal to the oracle; configurations A and B give bit-identical pages to the automatic
    choice. PreparedBatch.stats() equals the harness's plan of the shard (the plan the CPU suite checks)."""
    import torch
    ctxs, idx = contexts
    base = pe.edge_batches(edge)[batch]
    qs = rep(base)
    want = tile(want_pages(edge, batch, base, top_k))
    res = {}
    for name in ("auto", "A", "B"):
        res[name] = GpuIndexSearcher(idx[name]).search_batch(qs, RelevanceCollector(top_k, threshold))
    check(res["auto"], want, threshold, f"{batch} k={top_k} thr={threshold}")
    same(res["A"], res["auto"], f"{batch} k={top_k}: configuration A")
    same(res["B"], res["auto"], f"{batch} k={top_k}: configuration B")
    if threshold == THR and batch == "disj":
        assert (res["auto"].relation != 0).any(), "no query was pruned"
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    p = ph.plan(shard_dictionary(edge.shard), qs, top_k, threshold, sm_count=sm)
    pb = GpuIndexSearcher(idx["auto"]).prepare(qs, RelevanceCollector(top_k, threshold))
    try:
        st = pb.stats()
    finally:
        pb.close()
    assert st["work_items"] == p.n_work and st["alg_postings"] == p.alg_postings
    assert st["launches_per_run"] == 1 + int(p.n_probe_simple > 0) + int(p.n_probe_generic > 0)


@pytest.mark.parametrize("top_k", TOP_KS)
def test_search_after_inside_the_tie_group(contexts, edge, top_k):
    """Page 1 ends inside the tie group (equal scores across part and slice edges; the 16-way split query then runs a
    first-docs warm-up item with searchAfter); page 1 + page 2 is the 2k page, in both score modes and all configurations."""
    ctxs, idx = contexts
    q = pe.tie_query(edge)
    for thr in (THR, INT_MAX):
        full = want_pages(edge, "tie", [q], 2 * top_k)
        p1 = GpuIndexSearcher(idx["auto"]).search_batch(rep([q]), RelevanceCollector(top_k, thr))
        check(p1, tile(want_pages(edge, "tie", [q], top_k)), thr, f"tie page 1 k={top_k}")
        assert (p1.counts == top_k).all()
        last = ScoreDoc(int(p1.docs[0, top_k - 1]), float(p1.scores[0, top_k - 1]))
        assert (full[1][0, :2 * top_k] == np.float32(last.score)).sum() >= 2, "page 1 should end inside a tie"
        for name in ("auto", "A", "B"):
            p2 = GpuIndexSearcher(idx[name]).search_batch(rep([q]), RelevanceCollector(top_k, thr), search_after=[last] * REP)
            w2 = tile(want_pages(edge, "tie", [q], top_k, search_after=[last]))
            check(p2, w2, thr, f"tie page 2 k={top_k} {name}")
            for r in range(REP):
                n = int(p2.counts[r])
                assert np.array_equal(np.concatenate([p1.docs[r, :top_k], p2.docs[r, :n]]), full[0][0, :top_k + n])
                assert np.array_equal(np.concatenate([p1.scores[r, :top_k], p2.scores[r, :n]]).view(np.uint32),
                                      full[1][0, :top_k + n].view(np.uint32))


def test_three_leaves_with_doc_base(gpu_ctx, edge):
    """The same batches through GpuLeafSearcher over 3 leaves (doc_base 0, 300,001, 800,003: every leaf has its own
    partial granule and slice layout); pages equal the oracle's on the whole shard."""
    cuts = (0, 300_001, 800_003, pe.N_EDGE)
    leaves = [GpuIndex(gpu_ctx, edge.shard.doc_range(a, b)) for a, b in zip(cuts, cuts[1:])]
    ls = GpuLeafSearcher(gpu_ctx, leaves)
    try:
        assert [l.doc_base for l in leaves] == list(cuts[:3])
        for batch, qs in pe.edge_batches(edge).items():
            for k in (40, 512):
                for thr in (THR, INT_MAX):
                    check(ls.search_batch(rep(qs), RelevanceCollector(k, thr)), tile(want_pages(edge, batch, qs, k)), thr,
                          f"3 leaves {batch} k={k} thr={thr}")
    finally:
        ls.close()
        for l in leaves:
            l.close()


@pytest.mark.parametrize("threshold", [THR, INT_MAX], ids=["top_scores", "complete"])
def test_prepared_batch_reuse_across_deletes(contexts, edge, threshold):
    """One PreparedBatch planned without deletes (known hits, sweep warm-ups) runs twice bit-identically, then with deletes
    installed after prepare (the known hits are dropped), then with the deletes removed; each run equals the oracle of
    its live set."""
    ctxs, idx = contexts
    base = pe.edge_batches(edge)["disj"]
    qs = rep(base)
    k = 40
    live = np.ones(pe.N_EDGE, np.uint8)
    live[::7] = 0
    live[pe.TIE_STRIDE * 3::pe.TIE_STRIDE * 5] = 0
    live[pe.N_EDGE - 1] = 0
    gix = idx["auto"]
    pb = GpuIndexSearcher(gix).prepare(qs, RelevanceCollector(k, threshold))
    try:
        pb.run()
        r1 = pb.fetch()
        pb.run()
        r2 = pb.fetch()
        same(r1, r2, "second run of the same PreparedBatch")
        check(r1, tile(want_pages(edge, "disj", base, k)), threshold, "reuse: no deletes")
        gix.set_live_docs(live)
        pb.run()
        check(pb.fetch(), tile(want_pages(edge, "disj", base, k, live=live)), threshold, "reuse: deletes after prepare")
        gix.set_live_docs(None)
        pb.run()
        same(pb.fetch(), r1, "reuse: deletes removed")
    finally:
        gix.set_live_docs(None)
        pb.close()


_LINE = re.compile(r"\[nrtgpu probe (simple|generic)\] (\d+) items, .*?, ([\d.]+) runs/item \(([\d.]+) staged\).*?([\d.]+) flushes/item")


def probe_counters(capfd, gix, qs, k, thr):
    capfd.readouterr()
    GpuIndexSearcher(gix).search_batch(qs, RelevanceCollector(k, thr))
    err = capfd.readouterr().err
    out = {m.group(1): dict(items=int(m.group(2)), runs=float(m.group(3)), staged=float(m.group(4)), flushes=float(m.group(5)))
           for m in _LINE.finditer(err)}
    assert out, f"no probe counters on stderr: {err[-500:]}"
    return out


def test_kernel_counters_prove_the_edges_are_reached(contexts, edge, capfd):
    """Counters of the profiling instantiation: clustered items run several runs (one-granule runs beside a short list
    and a list searched in global memory), the stage limits split staged from global-memory short lists in
    configuration A (TOP_SCORES) and B (COMPLETE), and the tie batch flushes its candidate buffer."""
    ctxs, idx = contexts
    g = idx["dbg"]
    t = edge.term
    for qs in ([pe.disj(t["C0"], t["C1"], t["C2"], t["C3"])], [pe.disj(t["C0"], t["C1"], t["C2"], t["S_RUN"])],
               [pe.disj(t["C3"], t["C2"], t["C1"], t["SH_3969"])]):
        for thr in (THR, INT_MAX):
            c = probe_counters(capfd, g, qs, 40, thr)["simple"]
            assert c["runs"] > 2.0 and c["staged"] > 1.0, c
    c = probe_counters(capfd, g, [pe.bq((t["C0"], pe.Occur.MUST), (t["C1"], pe.Occur.MUST))], 40, INT_MAX)["generic"]
    assert c["runs"] > 1.5, c   # (two long lists: three cluster granules per run)
    # short lists alone (their slice-1 item holds all of the list): staged up to kShortMax, searched in place above it
    for L, thr, staged in ((3968, THR, True), (3969, THR, False), (2432, INT_MAX, True), (2433, INT_MAX, False)):
        c = probe_counters(capfd, g, [pe.disj(t[f"SH_{L}"])], 40, thr)["simple"]
        assert (c["staged"] > 0) == staged, (L, thr, c)
    # pairs whose sum meets or passes the limit: the first list is staged either way (the plan test shows the split)
    for a, b_, thr in (("1984", "1984b", THR), ("1984", "2000", THR), ("1216", "1216b", INT_MAX), ("1216", "1232", INT_MAX)):
        c = probe_counters(capfd, g, [pe.disj(t[f"SH_{a}"], t[f"SH_{b_}"])], 40, thr)["simple"]
        assert c["staged"] > 0, (a, b_, c)
    for thr in (THR, INT_MAX):
        c = probe_counters(capfd, g, [pe.tie_query(edge)], 512, thr)["simple"]
        assert c["flushes"] > 0 and c["items"] >= 3 * 16, c


def test_small_shard_planes_without_granule_rows(gpu_ctx):
    """Under 262,144 docs: planes without skip data (part bounds searched in their postings) beside planes with rows,
    split parts, in both score modes and all top_k."""
    b = pe.small_shard()
    qs = pe.small_batches(b)
    gix = GpuIndex(gpu_ctx, b.shard)
    try:
        for k in TOP_KS:
            for thr in (THR, INT_MAX):
                check(GpuIndexSearcher(gix).search_batch(rep(qs), RelevanceCollector(k, thr)), tile(want_pages(b, "small", qs, k)), thr,
                      f"small k={k} thr={thr}")
    finally:
        gix.close()
