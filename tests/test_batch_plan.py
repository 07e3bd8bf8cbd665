"""The host batch compiler and probe work planner (nrtsearch_b200/csrc/batch_plan.inc) on dictionaries alone, through the
g++ harness tests/csrc/plan_harness.cpp: the work list covers every (query, slice) exactly once, in the order the probe
kernel's queues expect, with sizes the kernels can index; the engine choice, driver selection, searchAfter keys and
known hit counts follow the documented rules; refusals keep their statuses and messages. Every item is read back
through the decoder the probe kernel uses, so planner and kernel cannot drift apart unseen. One GPU-marked test ties the
harness to the product: PreparedBatch.stats() of the engine equals the harness's plan on the same shards."""
import numpy as np
import pytest

import plan_harness as ph
from nrtsearch_b200 import _native
from nrtsearch_b200.search import BooleanQuery, BoostQuery, MatchAllDocsQuery, Occur, RangeQuery, ScoreDoc, TermQuery

INT_MAX = ph.INT_MAX
K = ph.constants()
ERR_INVALID, ERR_UNSUPPORTED = 1, 3   # include/nrtgpu.h NRTGPU_ERR_*


def disj(terms):
    q = BooleanQuery()
    for t in terms:
        q.add(TermQuery(int(t)), Occur.SHOULD)
    return q


def bq(*clauses, msm=0):
    q = BooleanQuery(minimum_number_should_match=msm)
    for c, o in clauses:
        q.add(TermQuery(int(c)) if isinstance(c, (int, np.integer)) else c, o)
    return q


def zipf_dict(rng, n_docs, n_terms=2000, deletes=False, max_x=None):
    """List lengths log-uniform over [1, n_docs / 2], the densest first-ish (a few lists above n_docs / 64 get planes,
    those of >= 4096 postings get granule rows)."""
    lens = np.minimum(n_docs, np.floor(10 ** rng.uniform(0, np.log10(max(n_docs / 2, 2)), n_terms))).astype(np.int64)
    off = np.zeros(n_terms + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    mx = rng.uniform(0.2, 3.0, n_terms).astype(np.float32) if max_x is None else max_x
    return ph.Dictionary(n_docs, off, term_max_x=mx, has_deletes=deletes, col_multi=np.array([0, 1], np.uint8),
                         col_n_distinct=np.array([1000, 0], np.int32))


def random_batch(rng, d, nq):
    qs = []
    for i in range(nq):
        n = int(rng.integers(1, 5))
        terms = rng.choice(d.n_terms, n, replace=False)
        shape = i % 6
        if shape < 3:
            qs.append(disj(terms))
        elif shape == 3:
            qs.append(bq(*[(t, Occur.MUST if j == 0 else Occur.SHOULD) for j, t in enumerate(terms)]))
        elif shape == 4:
            qs.append(bq(*[(t, Occur.SHOULD) for t in terms], (RangeQuery(0, 0, 500), Occur.FILTER)))
        else:
            qs.append(bq((MatchAllDocsQuery(), Occur.MUST), *[(t, Occur.SHOULD) for t in terms]))
    qs[7] = bq(*[(t, Occur.SHOULD) for t in rng.choice(d.n_terms, 2, replace=False)], msm=3)   # empty: msm > #SHOULD
    qs[nq // 2] = BooleanQuery()                                                                # empty: no clause
    return qs


def is_simple(q):
    """A query of the simple probe instantiation: a pure disjunction of scoring term clauses over one text field (no sort,
    no aggregations in these batches)."""
    return (q["single_field"] >= 0 and not q["has_nonterm"] and not q["nonterm_scoring"] and q["n_req"] == 0 and
            q["not_term_mask"] == 0 and q["msm"] <= 1 and not q["dense_driver"])


def check_plan(p, d):
    """Coverage, order and sizes of one probe plan on dictionary d (see the module docstring)."""
    pm, n_gran, gps = p.parts_max, p.n_gran, p.slice_docs // K["kGran"]
    assert pm & (pm - 1) == 0 and 1 <= pm <= 16
    assert p.n_lists == p.n_slices * pm + (1 if d.n_docs >= K["warm_min_docs"] else 0)
    for e in range(p.n_slices * pm + 2):
        assert 0 <= p.boundary_gran(e) <= n_gran
    assert p.n_probe_simple + p.n_probe_generic == p.n_work
    # warm-up items first; each segment slice-major; the simple segment holds exactly the simple queries' items
    flags = np.array([ph.decode(w)[3] for w in p.work_item])
    is_warm = (flags & (ph.ITEM_WARM_DOCS | ph.ITEM_SWEEP)) != 0
    n_warm = int(is_warm.sum())
    assert is_warm[:n_warm].all() and n_warm <= p.n_probe_simple
    assert n_warm == 0 or d.n_docs >= K["warm_min_docs"]
    for lo, hi in ((n_warm, p.n_probe_simple), (p.n_probe_simple, p.n_work)):
        sl = [ph.decode(w)[0] for w in p.work_item[lo:hi]]
        assert sl == sorted(sl), "items are not slice-major"
    simple = np.array([is_simple(q) for q in p.queries], bool)
    assert simple[p.work_query[:p.n_probe_simple]].all(), "a generic query's item in the simple segment"
    assert not simple[p.work_query[p.n_probe_simple:]].any(), "a simple query's item in the generic segment"
    # coverage: every non-empty query has items, and the parts of each of its (query, slice) pairs cover the slice's
    # granules exactly once (slice 0 from kWarmGran on behind a first-docs warm-up item)
    nonempty = {q for q in range(len(p.queries)) if not p.queries[q]["empty"]}
    assert set(p.work_query.tolist()) == nonempty, "a non-empty query without items, or an empty one with items"
    cover = {}
    sweep_q, docs_warm_q = set(), set()
    for q, w in zip(p.work_query.tolist(), p.work_item.tolist()):
        s, part, lp, f, slot = ph.decode(w)
        g_lo, g_hi, e_lo, e_hi, out = p.span(w)
        if f & ph.ITEM_SWEEP:
            sweep_q.add(q)
            assert out == p.n_lists - 1 and (e_lo, e_hi) == (0, p.n_slices * pm)
            continue
        if f & ph.ITEM_WARM_DOCS:
            docs_warm_q.add(q)
            assert s == 0 and g_lo == 0 and g_hi == min(K["kWarmGran"], gps, n_gran) and out == p.n_lists - 1
            assert e_hi == p.n_slices * pm + 1
            continue
        assert 0 <= out < p.n_slices * pm and part < (1 << lp)
        g_count = min(gps, n_gran - s * gps)
        c = cover.setdefault((q, s), np.zeros(g_count, np.int32))
        c[g_lo:g_hi] += 1
    assert not sweep_q & docs_warm_q
    g0 = min(gps, n_gran)   # granules of slice 0
    want = {(q, s) for q in nonempty for s in range(p.n_slices)
            if not (s == 0 and q in docs_warm_q and g0 <= K["kWarmGran"])}   # (slice 0 may be the warm-up item's alone)
    assert set(cover) == want, f"(query, slice) pairs without items: {sorted(want - set(cover))[:5]}"
    for (q, s), c in cover.items():
        start = min(K["kWarmGran"], len(c)) if (s == 0 and q in docs_warm_q) else 0
        assert (c[start:] == 1).all() and (c[:start] == 0).all(), f"query {q} slice {s}: granules not covered exactly once"
    return sweep_q, docs_warm_q


@pytest.mark.parametrize("seed", range(12))
def test_random_plans_cover_and_order(seed):
    """Random dictionaries (1K to 10M docs, with and without tf planes, granule rows and deletes) and random batches at
    both score modes and several top_k: coverage, order and sizes of every plan; sweep warm-up items only for queries
    without searchAfter, on their largest-bound list of at least 2 * top_k postings."""
    rng = np.random.default_rng(seed)
    n_docs = int(10 ** rng.uniform(3, 7))
    d = zipf_dict(rng, n_docs, deletes=bool(seed % 3 == 2))
    qs = random_batch(rng, d, 64)
    after = [ScoreDoc(int(rng.integers(0, n_docs)), 1.5) if i % 5 == 4 else None for i in range(len(qs))]
    for top_k, thr in ((10, 1000), (100, INT_MAX), (512, 2000)):
        p = ph.plan(d, qs, top_k, thr, search_after=after)
        assert not p.wide and p.n_slices == -(-n_docs // p.slice_docs)
        sweep_q, _ = check_plan(p, d)
        for q in sweep_q:
            assert after[q] is None
            w = p.work_item[(p.work_query == q) & np.array([bool(ph.decode(x)[3] & ph.ITEM_SWEEP) for x in p.work_item])][0]
            slot = ph.decode(w)[4]
            rec = p.queries[q]
            cl = p.clauses[rec["clause_begin"]:rec["clause_begin"] + rec["n_clauses"]]
            terms = cl[cl["kind"] == 0]
            lead = terms[terms["slot"] == slot][0]
            assert lead["ub"] == terms["ub"].max() and lead["n_post"] >= 2 * top_k


def test_large_shard_has_planes_rows_and_warm_ups():
    """10M docs: the dictionary has tf planes and granule rows, the plan has warm-up items of both kinds, parts, and
    more than one slice, and is still consistent."""
    rng = np.random.default_rng(99)
    d = zipf_dict(rng, 10_000_000, n_terms=20_000)
    tp, tg = ph.index_rules(d.n_docs, d.term_off)
    assert (tp >= 0).any() and (tg >= 0).any()
    lens = np.diff(d.term_off)
    dense, planes = lens * 64 >= d.n_docs, tp >= 0
    stride = (d.n_docs + 15) // 16 * 16 + 16
    assert (planes <= dense).all() and planes.sum() == min(dense.sum(), 1024, (8 << 30) // stride)   # the densest keep theirs
    assert lens[planes].min() >= lens[dense & ~planes].max()
    assert sorted(tp[planes].tolist()) == list(range(planes.sum()))
    assert ((lens >= 4096) == (tg >= 0)).all() and sorted(tg[tg >= 0].tolist()) == list(range((tg >= 0).sum()))
    qs = random_batch(rng, d, 256)
    qs += [disj([1, 2])]
    p = ph.plan(d, qs, 10, 1000)
    sweep_q, docs_warm_q = check_plan(p, d)
    assert p.n_slices == 20 and p.parts_max > 1 and sweep_q
    p = ph.plan(d, qs, 10, INT_MAX, search_after=[ScoreDoc(5, 2.0)] * len(qs))
    sweep_q, docs_warm_q = check_plan(p, d)
    assert not sweep_q and docs_warm_q


def test_engine_choice():
    """Wide exactly when a query has more than 4 term clauses or top_k > 512: one item per non-empty query and
    1,048,576-doc slice; the wide-only refusals of sorted search and aggregations keep their messages."""
    rng = np.random.default_rng(5)
    d = zipf_dict(rng, 2_500_000)
    narrow = [disj([1, 2, 3, 4]), bq((5, Occur.MUST), (6, Occur.SHOULD)), BooleanQuery()]
    assert not ph.plan(d, narrow, 512).wide
    for qs, k in ((narrow + [disj([1, 2, 3, 4, 5])], 10), (narrow, 513)):
        p = ph.plan(d, qs, k)
        assert p.wide and p.slice_docs == K["kWideSliceDocs"] == 1_048_576 and p.n_slices == 3
        assert p.n_work == 3 * (len(qs) - 1) and p.n_probe_simple == p.n_probe_generic == 0
        assert p.parts_max == 1 and p.n_lists == 3 and sorted(set(p.work_item.tolist())) == [0, 1, 2]
        with pytest.raises(ph.PlanError, match="sorted search: more than 4 term clauses or top_k > 512") as e:
            ph.plan(d, qs, k, sort=_native.Sort(1, 0, 0, 0, 0, None))
        assert e.value.rc == ERR_UNSUPPORTED
        with pytest.raises(ph.PlanError, match="aggregations: more than 4 term clauses") as e:
            ph.plan(d, qs, k, aggs=[_native.Aggregation(2, 0, 0, 0, 0, 0)])
        assert e.value.rc == ERR_UNSUPPORTED
    with pytest.raises(ph.PlanError, match="top_k > 1024"):
        ph.plan(d, narrow, 1025)


def test_refusals_keep_status_and_first_error():
    rng = np.random.default_rng(6)
    d = zipf_dict(rng, 100_000, n_terms=50)
    cases = [([disj(range(9))], 10, ERR_UNSUPPORTED, "more than 8 term clauses"),
             ([bq(*[(RangeQuery(0, 0, 1), Occur.FILTER)] * 17)], 10, ERR_UNSUPPORTED, "more than 16 clauses"),
             ([disj([50])], 10, ERR_INVALID, "term id out of range"),
             ([bq((RangeQuery(7, 0, 1), Occur.FILTER))], 10, ERR_INVALID, "column id out of range"),
             ([BoostQuery(disj([1]), 1.0)], 0, ERR_INVALID, "numHits must be > 0"),
             ([disj([50]), disj(range(9))], 10, ERR_INVALID, "term id out of range")]   # the first error of several
    for qs, k, rc, msg in cases:
        with pytest.raises(ph.PlanError, match=msg) as e:
            ph.plan(d, qs, k)
        assert e.value.rc == rc
    with pytest.raises(ph.PlanError, match="sorted searchAfter needs after_values"):
        ph.plan(d, [disj([1])], 10, sort=_native.Sort(1, 0, 0, 0, 0, None), search_after=[ScoreDoc(3, 1.0)])
    with pytest.raises(ph.PlanError, match="sort on a multi-valued column"):
        ph.plan(d, [disj([1])], 10, sort=_native.Sort(1, 1, 0, 0, 0, None))
    with pytest.raises(ph.PlanError, match="aggregation on a multi-valued column"):
        ph.plan(d, [disj([1])], 10, aggs=[_native.Aggregation(2, 1, 0, 0, 0, 0)])


def test_compilation_drivers_after_keys_known_hits():
    """Driver selection (the rarest required list, a dense driver for range-led and match-all, every SHOULD for pure
    disjunctions), `empty`, searchAfter keys for after_doc below, inside and above the leaf, and known_hits."""
    off = np.array([0, 100, 300, 1300, 1310], np.int64)   # lists of 100, 200, 1000, 10 postings
    d = ph.Dictionary(50_000, off, doc_base=1000, col_multi=np.zeros(1, np.uint8))
    qs = [disj([0, 1, 2]),                                                     # pure disjunction
          bq((2, Occur.MUST), (3, Occur.FILTER), (0, Occur.SHOULD)),          # rarest required: term 3 (slot 1)
          bq((RangeQuery(0, 0, 9), Occur.FILTER), (0, Occur.SHOULD)),         # range-led
          bq((MatchAllDocsQuery(), Occur.SHOULD), (1, Occur.SHOULD)),         # match-all
          bq((0, Occur.SHOULD), (1, Occur.SHOULD), msm=3),                    # empty: msm > #SHOULD
          bq((0, Occur.MUST_NOT)),                                            # empty: no required / SHOULD clause
          disj([0, 2]), disj([0, 2]), disj([0, 2])]
    after = [None] * 6 + [ScoreDoc(500, 2.0), ScoreDoc(1000 + 20, 2.0), ScoreDoc(1000 + 50_000, 2.0)]
    p = ph.plan(d, qs, 10, 100, search_after=after)
    q = p.queries
    assert q["driver_mask"][0] == 0b111 and not q["dense_driver"][0]
    assert q["driver_mask"][1] == 0b10 and q["has_non_driver"][1]
    assert q["dense_driver"][2] and q["dense_driver"][3]
    assert q["empty"][4] and q["empty"][5] and not q["empty"][:4].any()
    key = lambda s, doc: (int(np.float32(s).view(np.uint32)) | 0x80000000) << 32 | (~doc & 0xFFFFFFFF)
    assert q["after_key"][6] == (int(np.float32(2.0).view(np.uint32)) | 0x80000000) + 1 << 32   # every doc here follows
    assert q["after_key"][7] == key(2.0, 20)
    assert q["after_key"][8] == key(2.0, INT_MAX)                                           # every doc here precedes
    assert list(p.known_hits) == [1000, 0, 0, 0, 0, 0, 1000, 1000, 1000]   # simple queries only: the longest list
    d.has_deletes = True
    assert not ph.plan(d, qs, 10, 100, search_after=after).known_hits.any()


def test_hand_derived_plan():
    """A 300,000-doc shard and two queries at top_k 10, threshold 1000 (TOP_SCORES), written out by hand:
    q0 = SHOULD terms 0, 1, 2 (40,000 postings each, max_x 1.0, 2.0, 0.5); q1 = MUST term 3 (30,000) + SHOULD term 0.
    - Slices: at most 512 granules of 1024 docs, so one slice of ceil(300,000 / 1024) = 293 granules (300,032 docs).
      Warm-up items are on (300,000 >= 8 * 32 * 1024 docs), so there are n_slices * parts_max + 1 candidate lists.
    - q0 is a pure disjunction (simple). Its largest bound weight - weight / (1 + max_x) is term 1's (slot 1), whose
      40,000 postings are >= 2 * top_k: one sweep item, item_encode_sweep(1) = 1 << 16 | 4 << 24, no first-docs item.
      q1 has a required clause: generic, no warm-up.
    - Parts: cost q0 = 120,000, q1 = 70,000; postings per resident CTA = 190,000 / (3 * 132) = 479, so every item bound
      is the 32,768 floor. A pair splits while cost >> lp > 32,768 and 293 >> (lp + 1) >= 8: lp = 2 for both (q0:
      30,000 after two halvings; q1: 17,500). parts_max = 4, fine = ceil(293 / 4) = 74: granules [0, 74), [74, 148),
      [148, 222), [222, 293); part p writes list p, the sweep item list 4.
    - Order: the sweep item, q0's parts (simple), then q1's parts (generic)."""
    off = np.array([0, 40_000, 80_000, 120_000, 150_000], np.int64)
    d = ph.Dictionary(300_000, off, term_max_x=np.array([1.0, 2.0, 0.5, 1.0], np.float32))
    qs = [disj([0, 1, 2]), bq((3, Occur.MUST), (0, Occur.SHOULD))]
    p = ph.plan(d, qs, 10, 1000, sm_count=132)
    assert (p.n_slices, p.slice_docs, p.n_gran, p.parts_max, p.n_lists) == (1, 300_032, 293, 4, 5)
    sweep = 1 << 16 | 4 << 24
    want_w = [sweep] + [part << 16 | 2 << 20 for part in range(4)] * 2
    assert p.work_query.tolist() == [0] * 5 + [1] * 4 and p.work_item.tolist() == want_w
    assert (p.n_probe_simple, p.n_probe_generic) == (5, 4)
    assert [p.span(w)[:2] for w in want_w[1:5]] == [(0, 74), (74, 148), (148, 222), (222, 293)]
    assert p.span(sweep)[4] == 4 and [p.span(w)[4] for w in want_w[1:5]] == [0, 1, 2, 3]
    assert list(p.known_hits) == [40_000, 0] and p.alg_postings == 190_000


# ---------------------------------------------------------------- the harness against the product

def shard_dictionary(sh):
    """The planner's dictionary of a HostShard; term_max_x from numpy as max(float32(tf) * cache[norm]) per term."""
    n_terms = len(sh.term_off) - 1
    tf = np.zeros(n_terms, np.int32) if sh.term_field is None else np.asarray(sh.term_field, np.int32)
    term_of = np.repeat(np.arange(n_terms), np.diff(sh.term_off))
    x = np.zeros(len(sh.post_docs), np.float32)
    for f, fld in enumerate(sh.fields):
        avgdl = np.float32(fld.sum_total_term_freq / fld.doc_count) if fld.doc_count > 0 else np.float32(1.0)
        cache = ph.bm25_cache(fld.k1, fld.b, float(avgdl))
        sel = tf[term_of] == f
        norm = fld.norms[sh.post_docs[sel]] if fld.norms is not None else np.ones(int(sel.sum()), np.int64)
        x[sel] = np.asarray(sh.post_freqs[sel], np.float32) * cache[norm]
    mx = np.zeros(n_terms, np.float32)
    nz = np.diff(sh.term_off) > 0
    mx[nz] = np.maximum.reduceat(x, sh.term_off[:-1][nz])
    return ph.Dictionary(sh.n_docs, sh.term_off, term_field=tf, term_df=sh.term_df, term_max_x=mx,
                         field_doc_count=np.array([f.doc_count for f in sh.fields], np.int64), doc_base=sh.doc_base,
                         col_multi=np.zeros(len(sh.columns), np.uint8), has_deletes=sh.live_docs is not None)


@pytest.mark.gpu
def test_harness_plan_equals_product(gpu_ctx):
    """PreparedBatch.stats() (work_items, launches_per_run, alg_postings) of GpuIndexSearcher.prepare equals the
    harness's plan of the same shard: bench-shaped disjunctions on a multi-slice shard, a conjunction with a range,
    searchAfter, deletes and a wide batch."""
    import torch
    from nrtsearch_b200 import index as ix
    from nrtsearch_b200.search import GpuIndex, GpuIndexSearcher, RelevanceCollector
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    sh = ix.synth_text_shard(1_200_000, 50_000)
    sh.columns, sh.column_has = [ix.synth_int_column(sh.n_docs)], [None]
    terms = ix.synth_query_terms(256, 3, 50_000)
    bench = [disj(t) for t in terms]
    conj = [bq((int(t[0]), Occur.MUST), (int(t[1]), Occur.MUST), (RangeQuery(0, 100_000, 600_000), Occur.FILTER)) for t in terms[:64]]
    after = [ScoreDoc(int(i * 3001 % sh.n_docs), 3.0) for i in range(64)]
    wide = [disj(list(t) + [int(t[0]) + 1, int(t[1]) + 1]) for t in terms[:32]]
    live = np.ones(sh.n_docs, np.uint8)
    live[::11] = 0
    cases = [("bench", bench, 100, 1000, None, None), ("bench COMPLETE", bench, 100, INT_MAX, None, None),
             ("conj + range", conj, 10, 1000, None, None), ("searchAfter", bench[:64], 10, 1000, after, None),
             ("wide", wide, 10, 1000, None, None), ("deletes", bench + conj, 10, 1000, None, live)]
    gix = GpuIndex(gpu_ctx, sh)
    try:
        s = GpuIndexSearcher(gix)
        for what, qs, k, thr, sa, lv in cases:
            gix.set_live_docs(lv)
            sh.live_docs = lv
            b = s.prepare(qs, RelevanceCollector(k, thr), search_after=sa)
            try:
                got = b.stats()
            finally:
                b.close()
            p = ph.plan(shard_dictionary(sh), qs, k, thr, search_after=sa, sm_count=sm)
            launches = 1 + (int(p.n_work > 0) if p.wide else int(p.n_probe_simple > 0) + int(p.n_probe_generic > 0))
            want = {"work_items": p.n_work, "launches_per_run": launches, "alg_postings": p.alg_postings}
            assert got == want, f"{what}: product {got}, harness {want}"
    finally:
        sh.live_docs = None
        gix.close()
