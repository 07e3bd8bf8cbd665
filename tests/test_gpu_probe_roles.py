"""The MAXSCORE role counters of the profiling probe instantiation (NRTGPU_DEBUG_MODES): items that started without a
threshold and items whose roles went stale, in total and in slices 0 and 1. With no warm-up items
(NRTGPU_WARM_MIN_DOCS above the shard size) every query's first items start at theta = 0, so the counters must see
them; with warm-ups the pages are the same. Pages are checked against the exhaustive oracle in both score modes."""
import os
import re

import pytest

import oracle
from helpers import assert_same_hits
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import GpuContext, GpuIndex, GpuIndexSearcher, RelevanceCollector, compile_queries
import probe_edge_shards as pe

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
N_DOCS = 600_000             # two 512K-doc slices, above the warm-up minimum (262,144 docs)
TOP_K = 10

_ITEMS = re.compile(r"\[nrtgpu probe simple\] (\d+) items, ")
_ROLES = re.compile(r"\[nrtgpu probe simple\] roles: (\d+) items start without a threshold \(([\d.]+)% of item cycles; "
                    r"slice 0 (\d+), slice 1 (\d+)\); (\d+) items end with stale roles \(([\d.]+)% of item cycles, [\d.]+ cyc each, "
                    r"(\d+) driver postings, (\d+) in lists that turned non-essential; slice 0 (\d+), slice 1 (\d+)\)")


def _context(**env):
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
def setup(gpu_ctx):
    sh = ix.synth_text_shard(N_DOCS, 20_000)
    terms = ix.synth_query_terms(48, 3, 20_000, log10_lo=1.0, log10_hi=4.0)
    qs = [pe.disj(*(int(x) for x in t)) for t in terms]
    ctxs = {"warm": _context(NRTGPU_DEBUG_MODES="1"),
            "cold": _context(NRTGPU_DEBUG_MODES="1", NRTGPU_WARM_MIN_DOCS=str(4 * N_DOCS))}
    idx = {k: GpuIndex(c, sh) for k, c in ctxs.items()}
    carr, ncl, qarr, nq = compile_queries(qs)
    want = oracle.search_compiled(oracle.OracleIndex(sh), carr, ncl, qarr, nq, TOP_K)
    yield qs, idx, want
    for g in idx.values():
        g.close()
    for c in ctxs.values():
        c.close()


def run(capfd, gix, qs, thr):
    capfd.readouterr()
    r = GpuIndexSearcher(gix).search_batch(qs, RelevanceCollector(TOP_K, thr))
    err = capfd.readouterr().err
    items, roles = _ITEMS.search(err), _ROLES.search(err)
    assert items and roles, f"no role counters on stderr: {err[-500:]}"
    c = [float(x) if "." in x else int(x) for x in roles.groups()]
    return r, int(items.group(1)), dict(zip(("theta0", "theta0_pct", "theta0_s0", "theta0_s1", "stale", "stale_pct",
                                            "stale_post", "stale_turned", "stale_s0", "stale_s1"), c))


@pytest.mark.parametrize("threshold", [50, INT_MAX], ids=["top_scores", "complete"])
def test_role_counters_see_items_without_a_threshold(setup, capfd, threshold):
    qs, idx, want = setup
    for key in ("cold", "warm"):
        r, items, c = run(capfd, idx[key], qs, threshold)
        assert_same_hits((r.docs, r.scores, r.counts, r.total_hits, r.relation), want, what=f"{key} {threshold}")
        gte = r.relation != 0
        assert not (threshold == INT_MAX and gte.any()), f"{key}: COMPLETE reported GREATER_THAN_OR_EQUAL_TO"
        assert (r.total_hits[gte] > threshold).all() and (r.total_hits[gte] <= want[3][gte]).all(), f"{key}: lower bound"
        assert c["theta0_s0"] + c["theta0_s1"] <= c["theta0"] <= items, c
        assert c["stale_s0"] + c["stale_s1"] <= c["stale"] <= items, c
        assert 0.0 <= c["theta0_pct"] <= 100.0 and 0.0 <= c["stale_pct"] <= 100.0, c
        assert c["stale_turned"] <= c["stale_post"], c   # (a list that turned non-essential led the item)
        if key == "cold":   # no warm-up: the first item of every query starts at theta = 0, at least one per query
            assert c["theta0"] >= len(qs) and c["theta0_s0"] >= 1, c
