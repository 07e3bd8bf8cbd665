"""posting_probe_kernel at the boundaries of its rounds (kR * 256 = 512 driver postings each; the postings are fetched two
rounds ahead and the plane gathers issued one round ahead of the round that uses them): driver lists of 1, 511, 512,
513, 1023, 1024 and 1025 postings, each lying whole in one work item and one run of a pure disjunction, read from the stage (configuration A)
and in place from global memory (configuration B, where a short list of exactly the stage's short-list capacity is
staged first), probing a tf plane and a staged list; the same lists driving the generic instantiation and a dense sweep
with four probed slots; and candidate-buffer flushes inside a driver list at top_k 512. Every page is compared with the
exhaustive oracle (the edge-shard harness: tests/probe_edge_shards.py, tests/test_gpu_probe_edges.py)."""
import numpy as np
import pytest

import plan_harness as ph
import probe_edge_shards as pe
from test_batch_plan import shard_dictionary
from test_gpu_probe_edges import INT_MAX, THR, TOP_KS, _context, check, probe_counters, same, want_pages
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import GpuIndex, GpuIndexSearcher, Occur, RangeQuery, RelevanceCollector

N = pe.N_SMALL
ROUND_LENGTHS = (1, 511, 512, 513, 1023, 1024, 1025)
FILL = pe.K_SHORT_MAX["B"]   # staged whole in configuration B, so that a short list after it is searched and read in place


def round_shard() -> pe.Built:
    """200,003 docs (one slice): a plane without a granule row (P), a short list of FILL postings and the round-length
    short lists; every short list starts on a 16-posting boundary, so its staged segment is its own length rounded up."""
    rng = np.random.default_rng(512)
    im = pe._Image()
    d = pe._spread(0, N, -(-N // 64))
    im.add("P", d, pe._tf_cycle(d, 1))
    d = pe._spread(5, N - 3, FILL)
    im.add("FILL", d, pe._tf_cycle(d, 2), pbm=0)
    for L in ROUND_LENGTHS:
        d = pe._spread(L % 97, N - 1 - L % 89, L)
        im.add(f"RB_{L}", d, pe._tf_cycle(d, L), pbm=0)
    lens = rng.integers(2, 30, N)
    return im.shard(N, [ix.TextField(pe._BYTE4[lens], N, int(lens.sum()))], columns=[(np.arange(N) % 500).astype(np.int64)])


def round_batches(b: pe.Built) -> dict:
    t = b.term
    M, S, F = Occur.MUST, Occur.SHOULD, Occur.FILTER
    disj, bq = pe.disj, pe.bq
    rb = [t[f"RB_{L}"] for L in ROUND_LENGTHS]
    return {"disj": [disj(r) for r in rb] + [disj(r, t["P"]) for r in rb] + [disj(t["FILL"], r, t["P"]) for r in rb],
            "conj": [bq((r, M), (t["FILL"], S), (t["P"], S)) for r in rb] + [bq((t["FILL"], M), (r, M)) for r in rb],
            "dense": [bq((RangeQuery(0, 0, 499), F), (r, S), (t["P"], S), (t["FILL"], S), (t["RB_1"], S)) for r in rb[1:]]}


@pytest.fixture(scope="module")
def rounds():
    return round_shard()


@pytest.fixture(scope="module")
def indexes(gpu_ctx, rounds):
    """the shard's image in the default context and in contexts pinned to configurations A and B"""
    made = {"A": _context(NRTGPU_PROBE_CFG="1"), "B": _context(NRTGPU_PROBE_CFG="2")}
    idx = {k: GpuIndex(c, rounds.shard) for k, c in {"auto": gpu_ctx, **made}.items()}
    yield idx
    for g in idx.values():
        g.close()
    for c in made.values():
        c.close()


def test_round_lists_lie_whole_in_one_item(rounds):
    """(CPU) the pure disjunctions: one slice and no split parts, so every driver list is one run segment of its full
    length (the generic batches are split into parts, which cut the lists elsewhere)"""
    for thr in (THR, INT_MAX):
        p = ph.plan(shard_dictionary(rounds.shard), round_batches(rounds)["disj"], 512, thr, sm_count=132)
        assert p.n_slices == 1 and p.parts_max == 1 and p.n_probe_generic == 0, p.counters
        p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("threshold", [THR, INT_MAX], ids=["top_scores", "complete"])
@pytest.mark.parametrize("top_k", TOP_KS)
def test_round_boundaries_match_oracle(indexes, rounds, top_k, threshold):
    """Every batch page-for-page equal to the oracle, through configurations A and B and the automatic choice."""
    for batch, qs in round_batches(rounds).items():
        want = want_pages(rounds, "rounds_" + batch, qs, top_k)
        res = {k: GpuIndexSearcher(g).search_batch(qs, RelevanceCollector(top_k, threshold)) for k, g in indexes.items()}
        for k in ("auto", "A", "B"):
            check(res[k], want, threshold, f"{batch} k={top_k} thr={threshold} configuration {k}")
        same(res["A"], res["auto"], f"{batch} k={top_k}: configuration A")
        same(res["B"], res["auto"], f"{batch} k={top_k}: configuration B")


@pytest.mark.gpu
def test_flush_inside_a_driver_list(rounds, capfd):
    """top_k 512, ScoreMode.COMPLETE: the FILL list admits every doc it leads until the 1024-entry buffer is full, so the
    buffer is flushed part-way through the list and the sweep resumes after it; the page equals the oracle's."""
    t = rounds.term
    ctx = _context(NRTGPU_DEBUG_MODES="1")
    gix = GpuIndex(ctx, rounds.shard)
    try:
        for i, qs in enumerate(([pe.disj(t["FILL"], t["RB_1025"], t["P"])], [pe.disj(t["FILL"])], [pe.disj(t["RB_1025"])])):
            c = probe_counters(capfd, gix, qs, 512, INT_MAX)["simple"]
            assert c["flushes"] > 0, (i, c)
            check(GpuIndexSearcher(gix).search_batch(qs, RelevanceCollector(512, INT_MAX)), want_pages(rounds, f"flush_{i}", qs, 512),
                  INT_MAX, f"flush inside a driver list, query {i}")
    finally:
        gix.close()
        ctx.close()
