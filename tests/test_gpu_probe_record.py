"""The per-query record of posting_probe_kernel (DevProbeQuery: slot descriptors, the tf-pattern bound table, the
MAXSCORE order) on the queries that decide its contents: a pure disjunction whose first slot's term has no postings (an
absent list inside the bound table), four clauses with one term in two slots (equal bounds: the tie order of the MAXSCORE
prefix), lists of equal bounds from different terms, and an omitNorms field (no norms, no shortest length). Every page is
compared with the exhaustive oracle in both score modes, through configurations A and B and the automatic choice."""
import numpy as np
import pytest

import probe_edge_shards as pe
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import GpuIndex, GpuIndexSearcher, RelevanceCollector
from test_gpu_probe_edges import INT_MAX, THR, _context, check, same, want_pages

pytestmark = pytest.mark.gpu
N_DOCS = 1_000_003
REP = 24   # more work items than resident CTAs: most items start after their query's warm-up published a threshold


def record_shard():
    rng = np.random.default_rng(11)
    im = pe._Image()
    im.add("EMPTY", np.zeros(0, np.int64), np.zeros(0, np.int32))
    for name, df in (("DENSE", N_DOCS // 3), ("PLANE", N_DOCS // 40), ("LONG", 9000), ("SHORT", 700)):
        d = np.sort(rng.choice(N_DOCS, df, replace=False))
        im.add(name, d, pe._tf_cycle(d, df))
    twin = np.sort(rng.choice(N_DOCS - 1, 9000, replace=False))   # two lists of one tf per posting and one field length:
    im.add("TWIN_A", twin, np.full(len(twin), 2, np.int32))    # equal bounds from different terms
    im.add("TWIN_B", twin + 1, np.full(len(twin), 2, np.int32), pbm=5)
    for name, df in (("O_PLANE", N_DOCS // 30), ("O_SHORT", 900)):
        d = np.sort(rng.choice(N_DOCS, df, replace=False))
        im.add(name, d, pe._tf_cycle(d, df), fld=1)
    lens = rng.integers(2, 30, N_DOCS)
    lens[twin] = 7
    lens[twin + 1] = 7
    return im.shard(N_DOCS, [ix.TextField(pe._BYTE4[lens], N_DOCS, int(lens.sum())), ix.TextField(None, N_DOCS, 4 * N_DOCS)])


@pytest.fixture(scope="module")
def record():
    return record_shard()


def queries(b):
    t = b.term
    return [pe.disj(t["EMPTY"], t["DENSE"], t["SHORT"]), pe.disj(t["EMPTY"]), pe.disj(t["PLANE"], t["EMPTY"], t["LONG"], t["DENSE"]),
            pe.disj(t["PLANE"], t["SHORT"], t["PLANE"], t["DENSE"]), pe.disj(t["LONG"], t["LONG"], t["SHORT"], t["SHORT"]),
            pe.disj(t["TWIN_B"], t["TWIN_A"], t["DENSE"]), pe.disj(t["TWIN_A"], t["PLANE"], t["TWIN_B"], t["TWIN_A"]),
            pe.disj(t["O_PLANE"]), pe.disj(t["O_SHORT"], t["O_PLANE"]), pe.disj(t["O_PLANE"], t["O_SHORT"], t["O_PLANE"])]


@pytest.mark.parametrize("threshold", [THR, INT_MAX], ids=["top_scores", "complete"])
@pytest.mark.parametrize("top_k", [1, 40])
def test_record_queries_match_oracle_in_every_configuration(gpu_ctx, record, top_k, threshold):
    base = queries(record)
    qs = list(base) * REP
    want = tuple(np.concatenate([a] * REP) for a in want_pages(record, "record", base, top_k))
    made = {"A": _context(NRTGPU_PROBE_CFG="1"), "B": _context(NRTGPU_PROBE_CFG="2")}
    res = {}
    try:
        for name, ctx in {"auto": gpu_ctx, **made}.items():
            gix = GpuIndex(ctx, record.shard)
            try:
                res[name] = GpuIndexSearcher(gix).search_batch(qs, RelevanceCollector(top_k, threshold))
            finally:
                gix.close()
    finally:
        for c in made.values():
            c.close()
    check(res["auto"], want, threshold, f"record k={top_k} thr={threshold}")
    same(res["A"], res["auto"], f"record k={top_k}: configuration A")
    same(res["B"], res["auto"], f"record k={top_k}: configuration B")
    if threshold == THR:
        assert (res["auto"].relation != 0).any(), "no query was pruned"
