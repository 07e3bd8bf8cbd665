"""The structural edges the probe-kernel edge suite (tests/test_gpu_probe_edges.py) relies on, proved on the CPU: the
index-build rules give the lists of tests/probe_edge_shards.py the planes and granule rows their names claim, the list
layout reaches every alignment and both sides of both stage limits, the clusters fill the long-list reserve, and the work
planner (through the g++ harness) splits, drops and flags the work items as the suite's docstrings say. A shard or planner
change that moves a list off its edge fails here, not silently in the GPU suite."""
import numpy as np
import pytest

import plan_harness as ph
import probe_edge_shards as pe
from nrtsearch_b200.search import ScoreDoc
from test_batch_plan import check_plan, shard_dictionary

K = ph.constants()
INT_MAX = ph.INT_MAX
SM = 132   # H100 SXM


def seg_n(a, b, pbm):
    """probe_kernel.cuh seg_n: postings of the 16-aligned copy of list-relative postings [a, b)."""
    return 0 if b <= a else ((b + pbm + 15) & ~15) - ((a + pbm) & ~15)


@pytest.fixture(scope="module")
def edge():
    b = pe.edge_shard()
    return b, shard_dictionary(b.shard)


@pytest.fixture(scope="module")
def small():
    b = pe.small_shard()
    return b, shard_dictionary(b.shard)


def kinds(b, d):
    """name -> 'plane' / 'long' / 'short' (the kernel's kPlane / kLong / kShort-or-kGlobal) from the index-build rules."""
    tp, tg = ph.index_rules(d.n_docs, d.term_off)
    out = {}
    for name, t in b.term.items():
        out[name] = "plane" if tp[t] >= 0 else "long" if tg[t] >= 0 else "short"
    return out, tp, tg


def test_index_rule_edges(edge, small):
    """Plane at df * 64 >= n (df = ceil(n / 64) has one, one less has none), granule row at df >= 4096 (4096 has one,
    4095 none); the clusters are long lists; on the small shard lists of df ceil(n / 64) .. 4095 are planes without a
    granule row, and no list can be a long list (a row needs df >= 4096 > n / 64): a multi-run item never arises there,
    so the planes-without-rows are searched through the part boundaries (slice_bounds_kernel) only."""
    b, d = edge
    k, tp, tg = kinds(b, d)
    n = d.n_docs
    assert b.shard.df(b.term["P_HI"]) * 64 >= n > (b.shard.df(b.term["P_LO"])) * 64
    assert k["P_HI"] == "plane" and k["P_LO"] == "long" and k["G_HI"] == "long" and k["G_LO"] == "short"
    assert k["D0"] == k["D1"] == k["O_PLANE"] == "plane"
    assert all(k[f"C{i}"] == "long" for i in range(4)) and k["O_LONG"] == k["T_TIGHT"] == "long"
    assert all(k[x] == "short" for x in ("S_RUN", "T_TIE", "E_EDGES", "R_RARE", "S_WARM", "O_SHORT"))
    assert all(v == "short" for x, v in k.items() if x.startswith("SH_") or x.startswith("A"))
    sb, sd = small
    k2, tp2, tg2 = kinds(sb, sd)
    assert sd.n_docs < 262_144
    assert tp2[sb.term["PL_MIN"]] >= 0 and tg2[sb.term["PL_MIN"]] < 0 and sb.shard.df(sb.term["PL_MIN"]) == -(-sd.n_docs // 64)
    assert tp2[sb.term["PL_NOROW"]] >= 0 and tg2[sb.term["PL_NOROW"]] < 0 and sb.shard.df(sb.term["PL_NOROW"]) == 4095
    assert tp2[sb.term["PL_ROW"]] >= 0 and tg2[sb.term["PL_ROW"]] >= 0
    assert tp2[sb.term["BELOW"]] < 0 and tg2[sb.term["BELOW"]] < 0
    assert not ((tg2 >= 0) & (tp2 < 0)).any(), "a long list on a shard under 262,144 docs"


def test_alignment_and_stage_limits(edge):
    """The A lists start at all 16 residues of post_base mod 16 and the last of them ends the image with doc n - 1
    (its staged copy reads into the padding); the SH lists start 16-aligned, so their staged size is the length rounded up
    to 16 and they sit on both sides of kShortMax in both configurations, alone and in pairs."""
    b, d = edge
    res = sorted(b.post_base[f"A{i}"] % 16 for i in range(16))
    assert res == list(range(16))
    last = b.term["A15"]
    assert last == d.n_terms - 1 and b.shard.post_docs[-1] == d.n_docs - 1
    assert seg_n(0, b.shard.df(last), b.post_base["A15"] % 16) > b.shard.df(last)   # the copy passes the image's end
    need = {L: seg_n(0, b.shard.df(b.term[f"SH_{L}"]), b.post_base[f"SH_{L}"] % 16)
            for L in (2431, 2432, 2433, 3967, 3968, 3969, 1216, 1232, 1984, 2000)}
    A, B = pe.K_SHORT_MAX["A"], pe.K_SHORT_MAX["B"]
    assert (A, B) == (3968, 2432)
    assert need[2431] <= B and need[2432] == B and need[2433] > B and need[2433] <= A
    assert need[3967] <= A and need[3968] == A and need[3969] > A and need[2431] <= A
    assert need[1216] * 2 == B and need[1216] + need[1232] > B
    assert need[1984] * 2 == A and need[1984] + need[2000] > A
    assert b.post_base["SH_1216b"] % 16 == b.post_base["SH_1984b"] % 16 == 0
    # one work item holds the whole list: every posting in slice 1
    for name in [x for x in b.term if x.startswith("SH_")]:
        docs = b.shard.post_docs[b.shard.term_off[b.term[name]]:b.shard.term_off[b.term[name] + 1]]
        assert (docs // pe.SLICE_DOCS == 1).all()


def test_clusters_fill_the_long_list_reserve(edge):
    """Every cluster granule holds 1024 postings of each of C0..C3 (the partial last granule: its 723 docs): one granule of
    the four fits the long-list reserve 4 x (1024 + 32), two granules exceed either stage -- runs of one granule."""
    b, d = edge
    sh = b.shard
    n_gran = -(-d.n_docs // pe.GRAN)
    assert n_gran == 1221 and d.n_docs % pe.GRAN == 723 and d.n_docs % 4 == 3
    for i in range(4):
        t = b.term[f"C{i}"]
        docs = sh.post_docs[sh.term_off[t]:sh.term_off[t + 1]]
        cnt = np.bincount(docs // pe.GRAN, minlength=n_gran)
        assert set(np.nonzero(cnt)[0].tolist()) == set(pe.CLUSTER_GRANS)
        assert (cnt[pe.CLUSTER_GRANS[:-1]] == 1024).all() and cnt[1220] == 723
    for g in (24, 405, 406):   # consecutive cluster granules
        one = sum(seg_n(1024 * j, 1024 * (j + 1), b.post_base[f"C{i}"] % 16) for i in range(4)
                  for j in [pe.CLUSTER_GRANS.index(g)])
        two = sum(seg_n(1024 * j, 1024 * (j + 2), b.post_base[f"C{i}"] % 16) for i in range(4)
                  for j in [pe.CLUSTER_GRANS.index(g)])
        assert one <= 4 * (1024 + 32) < 6656 and two > 8192
    # S_RUN: postings in every cluster granule (in every run of an item over the clusters)
    t = b.term["S_RUN"]
    g = set((sh.post_docs[sh.term_off[t]:sh.term_off[t + 1]] // pe.GRAN).tolist())
    assert g == set(pe.CLUSTER_GRANS)


def test_doc_level_edges(edge):
    """Postings on both sides of every granule and slice edge and at n - 1; tf 1, 2, 3, 254, 255, > 255 in plane lists, in
    searched (long and short) lists and in the lists that lead; the shortest field length is held by T_TIGHT docs with
    every tf class; the tie group spans part edges (26-granule parts) and the slice 0/1 edge with equal norms."""
    b, d = edge
    sh, n = b.shard, d.n_docs
    lst = lambda x: (sh.post_docs[sh.term_off[b.term[x]]:sh.term_off[b.term[x] + 1]],
                     sh.post_freqs[sh.term_off[b.term[x]]:sh.term_off[b.term[x] + 1]])
    e, _ = lst("E_EDGES")
    g = np.arange(1, -(-n // pe.GRAN))
    assert np.isin(g * pe.GRAN - 1, e).all() and np.isin(g * pe.GRAN, e).all() and n - 1 in e and 0 in e
    for x in ("D0", "D1", "P_HI", "G_HI", "G_LO", "T_TIGHT", "E_EDGES"):
        assert set(pe.TFS.tolist()) <= set(lst(x)[1].tolist()), x
    for x in ("C0", "C1"):
        docs, f = lst(x)
        assert (f[docs % pe.GRAN == pe.GRAN - 1] >= 3).all()
    norms = sh.fields[0].norms
    nmin = norms[norms > 0].min()
    td, tf = lst("T_TIGHT")
    at_min = norms[td] == nmin
    assert (np.nonzero(norms == nmin)[0] == np.sort(td[at_min])).all()
    assert {1, 2, 3, 255, 256, 300} <= set(tf[at_min].tolist())
    tie, tf = lst("T_TIE")
    grp = tie[tf == 1]
    assert len(np.unique(norms[grp])) == 1 and len(grp) == 2000
    fine = 26 * pe.GRAN
    assert grp.min() < fine < grp.max() and grp.min() < pe.SLICE_DOCS < grp.max()
    assert len(np.unique(grp // fine)) >= 16


def items(p, q):
    out = []
    for w in p.work_item[p.work_query == q].tolist():
        s, part, lp, f, slot = ph.decode(w)
        out.append((s, part, lp, f, p.span(w)))
    return out


@pytest.mark.parametrize("top_k", [1, 40, 512])
@pytest.mark.parametrize("threshold", [50, INT_MAX])
def test_plan_of_the_edge_batches(edge, top_k, threshold):
    """3 slices of 407 granules, 16 parts of fine = 26 < kWarmGran granules. The heavy query (> 1.57M postings, rarest
    list of 30 postings) is split 16 ways; at top_k >= 40 it has a first-docs warm-up item (kItemWarmDocs), its part 0
    of slice 0 lies inside the warm-up granules and is dropped, and part 1 starts at granule 32 through kItemBehindWarm;
    at top_k 1 it has a sweep item instead. The omitNorms disjunctions run in the simple instantiation, conjunctions and
    range-led / match-all queries in the generic one (range-led and match-all with a dense driver)."""
    b, d = edge
    bt = pe.edge_batches(b)
    for name, qs in bt.items():
        p = ph.plan(d, qs, top_k, threshold, sm_count=SM)
        check_plan(p, d)
        assert (p.n_slices, p.slice_docs, p.n_gran) == (3, pe.SLICE_DOCS, 1221)
        if name == "disj":
            assert p.parts_max == 16 and -(-407 // p.parts_max) == 26 < K["kWarmGran"]
            assert (p.queries["single_field"] >= 0).all() and p.n_probe_generic == 0
            hq = next(i for i, q in enumerate(qs) if q == pe.heavy_query(b))
            it = items(p, hq)
            flags = [f for _, _, _, f, _ in it]
            assert all(lp == 4 for _, _, lp, f, _ in it if not f & (ph.ITEM_WARM_DOCS | ph.ITEM_SWEEP))
            s0 = sorted(part for s, part, _, f, _ in it if s == 0 and not f & (ph.ITEM_WARM_DOCS | ph.ITEM_SWEEP))
            if top_k == 1:
                assert any(f & ph.ITEM_SWEEP for f in flags) and s0 == list(range(16))
            else:
                assert any(f & ph.ITEM_WARM_DOCS for f in flags)
                assert s0 == list(range(1, 16)), "part 0 of slice 0 lies in the warm-up granules and is dropped"
                p1 = [sp for s, part, _, f, sp in it if s == 0 and part == 1][0]
                assert [f for s, part, _, f, _ in it if s == 0 and part == 1][0] & ph.ITEM_BEHIND_WARM
                assert p1[:2] == (32, 52)
            omit = [i for i, q in enumerate(qs) if all(b.shard.term_field[c.query.term] == 1 for c in q.clauses)]
            assert len(omit) == 4 and (p.queries["single_field"][omit] == 1).all()
        elif name == "conj":
            assert p.n_probe_simple == 0 and not p.queries["dense_driver"].any()
        else:
            assert p.n_probe_simple == 0 and p.queries["dense_driver"].all()
        if name == "disj":   # the other disjunctions of >= 2 * top_k postings warm up with a sweep item
            assert any(ph.decode(w)[3] & ph.ITEM_SWEEP for w in p.work_item)


def test_plan_of_search_after_in_the_tie_group(edge):
    """searchAfter pages of the tie query (split 16 ways): a first-docs warm-up item replaces the sweep, part 0 of slice 0
    is dropped and part 1 starts behind the warm-up granules -- searchAfter, split parts and a warm-up item together."""
    b, d = edge
    q = pe.tie_query(b)
    for k in (1, 40, 512):
        p = ph.plan(d, [q], k, 50, search_after=[ScoreDoc(5000 * pe.TIE_STRIDE, 1.0)], sm_count=SM)
        check_plan(p, d)
        it = items(p, 0)
        assert not any(f & ph.ITEM_SWEEP for _, _, _, f, _ in it)
        assert any(f & ph.ITEM_WARM_DOCS for _, _, _, f, _ in it)
        s0 = [(part, f, sp) for s, part, _, f, sp in it if s == 0 and not f & ph.ITEM_WARM_DOCS]
        assert [x[0] for x in s0] == list(range(1, 16)) and all(f & ph.ITEM_BEHIND_WARM for _, f, _ in s0)
        assert s0[0][2][:2] == (32, 52)


def test_plan_of_the_small_shard(small):
    """One slice, no warm-up items (n < 8 x 32 x 1024), the heaviest query split into parts: the planes without granule
    rows get their part bounds from a search of the postings."""
    b, d = small
    qs = pe.small_batches(b)
    for k, thr in ((1, 50), (40, INT_MAX), (512, 50)):
        p = ph.plan(d, qs, k, thr, sm_count=SM)
        check_plan(p, d)
        assert p.n_slices == 1 and p.parts_max >= 4 and p.n_lists == p.parts_max
        assert not any(ph.decode(w)[3] for w in p.work_item)
