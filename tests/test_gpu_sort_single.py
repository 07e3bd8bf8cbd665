"""The one-field sorted search (nrtgpu_search_sorted: TopFieldCollector over one numeric column or the doc id) against its
two references, oracle.search_sorted and the one-field Sorts of sort_fields_reference.search_sorted_fields (pinned to each
other on the CPU by tests/test_sort_single_reference.py; every Sort and page walk here is checked against both, the after
FieldDocs and the leaf merges against the oracle), bit-exact on docs, FieldDoc values (NaN and -0 bits included),
counts and EQUAL_TO totals. Every case also runs through nrtgpu_search_sorted_fields with a one-field order, which must
answer byte for byte the same.

The shard (tests/sort_single_shard.py): 1.1M docs at doc_base 5,000 in three probe slices, 8 % deleted, a 3,000-doc tie
group across the first slice edge, and columns whose missing value is held (int32 with INT32_MIN / MAX) or held by no
doc (int64 without Long.MIN / MAX, float without -inf, double without +-inf, a single-valued and an empty column). Cases:
every Sort at top_k 1 / 40 / 512; page walks at k = 97 whose boundaries land inside the group of docs without a value,
inside the tie group and at every value boundary; after FieldDocs below, between, above the held values and equal to the
missing value, with after_doc below, inside and above the leaf; three doc_range leaves merged by (value, global doc);
deletes installed and removed; terminateAfter and an expired deadline; every refusal. The index-time codes themselves
are checked through the test-only harness (tests/csrc/sort_code_harness.cu) against numpy."""
import copy
import ctypes as C

import numpy as np
import pytest

import oracle
import plan_harness as ph
import sort_code_harness as sch
import sort_single_shard as ss
from nrtsearch_b200 import _native
from nrtsearch_b200._native import SearchLimits, Sort as CSort
from nrtsearch_b200.search import FieldDoc, GpuIndex, GpuIndexSearcher, ScoreDoc, SortFieldCollector, SortType, compile_queries

pytestmark = pytest.mark.gpu

N, DOC_BASE = 1_100_000, 5_000
SLICE_DOCS = 359 * 1024   # 1075 granules of 1024 docs in 3 probe slices
TIE_LO = SLICE_DOCS - ss.TIE_DOCS // 2
K_WALK, WALK_PAGES, WALK_ALL = 97, 12, 5_000
REF_K = 6_000
SORTS = ss.sorts()
AFTER_QUERIES = [0, 1, 4, ss.ONLY_MISSING, 9]
AFTER_DOCS = [DOC_BASE - 7, DOC_BASE + TIE_LO + 1_500, DOC_BASE + 1_234, DOC_BASE + N + 9]   # below, inside (x2), above
CUTS = [0, 300_000, 700_000, N]
INVALID, UNSUPPORTED = 1, 3


@pytest.fixture(scope="module")
def setup(gpu_ctx):
    sh = ss.make_shard(N, DOC_BASE, TIE_LO)
    gix = GpuIndex(gpu_ctx, sh)
    yield sh, gix, oracle.OracleIndex(sh), {}
    gix.close()


def full_ref(setup, st):
    """the reference order of every query under st, the first REF_K hits, the same from both references; cached per Sort"""
    sh, _, oix, cache = setup
    key = ss.sort_id(st)
    if key not in cache:
        w = ss.want_fields(sh, ss.QUERIES, REF_K, st, oix=oix)
        wo = ss.want_oracle(sh, ss.QUERIES, REF_K, st, oix=oix)
        assert all(np.array_equal(a, b) for a, b in zip(w, wo)), "the two references differ"
        cache[key] = w
    return cache[key]


def both(s, qs, k, st, after=None):
    """nrtgpu_search_sorted, checked byte for byte against nrtgpu_search_sorted_fields with the one-field order [st]"""
    one = s.search_sorted(qs, SortFieldCollector(k, st), search_after=after)
    many = s.search_sorted(qs, SortFieldCollector(k, [st]), search_after=after)
    assert np.array_equal(one.counts, many.counts) and np.array_equal(one.total_hits, many.total_hits)
    assert np.array_equal(one.relation, many.relation)
    for q in range(len(qs)):
        n = one.counts[q]
        assert np.array_equal(one.docs[q, :n], many.docs[q, :n]), (ss.sort_id(st), q)
        assert np.array_equal(one.sort_values[q, :n], many.sort_values[q, :n, 0]), (ss.sort_id(st), q)
    return one


def assert_page(res, w, k, what):
    wd, wv, wc, wt = w
    assert np.array_equal(res.counts, np.minimum(wc, k)), what
    assert np.array_equal(res.total_hits, wt) and not res.relation.any(), what
    for q in range(len(res.counts)):
        n = res.counts[q]
        assert np.array_equal(res.docs[q, :n], wd[q, :n]), (what, q, res.docs[q, :6], wd[q, :6])
        assert np.array_equal(res.sort_values[q, :n], wv[q, :n]), (what, q)


def test_plan_has_slices_and_split_items(setup):
    """a sorted batch on this shard runs in at least 2 probe slices with split (query, slice) pairs, and the tie group
    straddles the first slice edge (the CPU planner on this dictionary)"""
    sh, _, _, _ = setup
    d = ph.Dictionary(N, sh.term_off, doc_base=DOC_BASE, col_multi=np.array([c == ss.C_MV for c in range(len(sh.columns))], np.uint8),
                      has_deletes=True)
    st = SortType(ss.C_F32, True, True, "float")
    p = ph.plan(d, ss.QUERIES, 40, sort=CSort(1, ss.C_F32, 1, 0, st.missing_value(), None))
    try:
        assert p.n_slices >= 2 and p.slice_docs == SLICE_DOCS and p.parts_max > 1
        assert max(ph.decode(w)[2] for w in p.work_item) > 0, "no (query, slice) pair was split"
        assert p.threshold == ph.INT_MAX
    finally:
        p.close()
    assert TIE_LO < SLICE_DOCS < TIE_LO + ss.TIE_DOCS


@pytest.mark.parametrize("st", SORTS, ids=ss.sort_id)
def test_every_sort(setup, st):
    sh, gix, oix, _ = setup
    w = full_ref(setup, st)
    wo = ss.want_oracle(sh, ss.QUERIES, 512, st, oix=oix)
    s = GpuIndexSearcher(gix)
    for k in (1, 40, 512):
        res = both(s, ss.QUERIES, k, st)
        assert_page(res, w, k, f"{ss.sort_id(st)} k={k} fields reference")
        assert_page(res, wo, k, f"{ss.sort_id(st)} k={k} oracle")


def walk(s, st, w, qids, qs=ss.QUERIES):
    """pages of k = 97, each after the last FieldDoc of the previous one: to the end under WALK_ALL matches, else 12
    pages; the concatenation equals the reference order, with no gap and no overlap"""
    wd, wv, _, wt = w
    goal = {q: int(wt[q]) if wt[q] <= WALK_ALL else K_WALK * WALK_PAGES for q in qids}
    got = {q: ([], []) for q in qids}
    after = {q: None for q in qids}
    active = [q for q in qids if goal[q] > 0]
    while active:
        aft = [after[q] for q in active]
        res = both(s, [qs[q] for q in active], K_WALK, st, None if all(a is None for a in aft) else aft)
        nxt = []
        for i, q in enumerate(active):
            assert res.total_hits[i] == wt[q] and not res.relation[i], (ss.sort_id(st), q)
            n = int(res.counts[i])
            got[q][0].extend(res.docs[i, :n].tolist())
            got[q][1].extend(res.sort_values[i, :n].tolist())
            assert n == K_WALK or len(got[q][0]) == wt[q], (ss.sort_id(st), q, "a short page before the end")
            if n == K_WALK and len(got[q][0]) < goal[q]:
                after[q] = FieldDoc(int(res.docs[i, n - 1]), int(res.sort_values[i, n - 1]))
                nxt.append(q)
        active = nxt
    for q in qids:
        docs, vals = got[q]
        assert len(docs) >= goal[q]
        assert docs == wd[q, :len(docs)].tolist(), (ss.sort_id(st), q, "pages differ from the reference order")
        assert vals == wv[q, :len(vals)].tolist(), (ss.sort_id(st), q)


@pytest.mark.parametrize("st", SORTS, ids=ss.sort_id)
def test_page_walks(setup, st):
    _, gix, _, _ = setup
    walk(GpuIndexSearcher(gix), st, full_ref(setup, st), [q for q in range(len(ss.QUERIES)) if q != ss.EMPTY])


@pytest.mark.parametrize("st", SORTS, ids=ss.sort_id)
def test_synthetic_afters(setup, st):
    sh, gix, oix, _ = setup
    qs, after = ss.synthetic_afters(sh, st, [ss.QUERIES[q] for q in AFTER_QUERIES], AFTER_DOCS)
    assert_page(both(GpuIndexSearcher(gix), qs, 40, st, after), ss.want_oracle(sh, qs, 40, st, after, oix), 40, ss.sort_id(st))


@pytest.fixture(scope="module")
def leaves(setup, gpu_ctx):
    sh = setup[0]
    out = [GpuIndex(gpu_ctx, sh.doc_range(a, b)) for a, b in zip(CUTS, CUTS[1:])]
    assert all(g.doc_base == DOC_BASE + a for g, a in zip(out, CUTS))
    yield out
    for g in out:
        g.close()


@pytest.mark.parametrize("st", SORTS, ids=ss.sort_id)
def test_three_leaves_merge_to_the_whole_reader(setup, leaves, st):
    """each leaf searched with the same after FieldDoc (after_doc in leaf 0, 1 or 2: below, inside and above every leaf)
    and the leaf pages merged by (value, global doc) equal the whole reader's page"""
    sh, _, oix, _ = setup
    k = 40
    docs = [DOC_BASE + (a + b) // 2 for a, b in zip(CUTS, CUTS[1:])]
    qs, after = ss.synthetic_afters(sh, st, [ss.QUERIES[q] for q in (0, 4, ss.ONLY_MISSING, 9)], docs)
    pages = [both(GpuIndexSearcher(g), qs, k, st, after) for g in leaves]
    wd, wv, wc, wt = ss.want_oracle(sh, qs, k, st, after, oix)
    assert np.array_equal(sum(p.total_hits for p in pages), wt)
    for q in range(len(qs)):
        md, mv = ss.merge_pages(st, [(p.docs[q], p.sort_values[q], p.counts[q]) for p in pages], k)
        assert md.tolist() == wd[q, :wc[q]].tolist(), (ss.sort_id(st), q, after[q])
        assert mv.tolist() == wv[q, :wc[q]].tolist(), (ss.sort_id(st), q)


def test_deletes_installed_and_removed(setup):
    """pages follow new deletes and their removal; the index-time codes stay as they were built"""
    sh, gix, _, _ = setup
    s = GpuIndexSearcher(gix)
    picks = [SortType(ss.C_F32, True, True, "float"), SortType(ss.C_I64, False, False, "long"), SortType(ss.C_I32, False, False, "int"),
             SortType("docid", True)]
    walked = [0, ss.ONLY_MISSING, 7, 9]
    try:
        for live in ((np.random.default_rng(8).random(N) >= 0.3).astype(np.uint8), None):
            sh2 = copy.copy(sh)
            sh2.live_docs = live
            oix2 = oracle.OracleIndex(sh2)
            gix.set_live_docs(live)
            for st in picks:
                w = ss.want_fields(sh2, ss.QUERIES, REF_K, st, oix=oix2)
                assert_page(both(s, ss.QUERIES, 512, st), w, 512, f"{ss.sort_id(st)} deletes {live is not None}")
                walk(s, st, w, walked)
    finally:
        gix.set_live_docs(sh.live_docs)
    st = picks[0]
    assert_page(both(s, ss.QUERIES, 40, st), full_ref(setup, st), 40, "deletes restored")


def raw_sorted(gix, qs, k, sort, lim=None, after_docs=None):
    """nrtgpu_search_sorted with every output: (status, docs, values, counts, totals, relation, hit_timeout, terminated)"""
    sd = None if after_docs is None else [ScoreDoc(d, 0.0) for d in after_docs]
    carr, ncl, qarr, nq = compile_queries(qs, sd)
    docs, vals = np.zeros((nq, k), np.int32), np.zeros((nq, k), np.int64)
    cnt, tot, rel, to, te = (np.zeros(nq, t) for t in (np.int32, np.int64, np.uint8, np.uint8, np.uint8))
    rc = _native.gpu_lib().nrtgpu_search_sorted(gix.handle, carr, ncl, qarr, nq, k, 0, None if sort is None else C.byref(sort),
                                                None if lim is None else C.byref(lim), None, docs.ctypes.data, vals.ctypes.data,
                                                cnt.ctypes.data, tot.ctypes.data, rel.ctypes.data, to.ctypes.data, te.ctypes.data)
    return rc, docs, vals, cnt, tot, rel, to, te


def test_limits(setup):
    sh, gix, _, _ = setup
    st = SortType(ss.C_F32, True, True, "float")
    sort = CSort(1, ss.C_F32, 1, 0, st.missing_value(), None)
    rc, docs, vals, cnt, tot, rel, to, te = raw_sorted(gix, ss.QUERIES, 40, sort, SearchLimits(0.0, 0.0, 0, 100, 0))
    assert rc == 0
    assert te[ss.MATCH_ALL] == 1 and rel[ss.MATCH_ALL] == 1   # match-all: far more than 100 matches
    assert te[7] == 0 and rel[7] == 0 and tot[7] == ss.EXACT_K   # 40 matches: not terminated
    rc, docs, vals, cnt, tot, rel, to, te = raw_sorted(gix, ss.QUERIES, 40, sort, SearchLimits(0.5, 1.0, 0, 0, 0))
    assert rc == 0   # the request spent its budget before the call: partial results
    assert to[ss.MATCH_ALL] == 1 and rel[ss.MATCH_ALL] == 1


def test_refusals(setup):
    sh, gix, _, _ = setup
    qs = ss.QUERIES[:2]
    ok = CSort(1, ss.C_I32, 0, 0, ss.I32_MIN, None)
    assert raw_sorted(gix, qs, 40, ok)[0] == 0
    assert raw_sorted(gix, qs, 513, ok)[0] == UNSUPPORTED                          # a wide batch
    assert raw_sorted(gix, qs, 40, CSort(1, ss.C_MV, 0, 0, 0, None))[0] == UNSUPPORTED   # a multi-valued column
    assert raw_sorted(gix, qs, 40, ok, after_docs=[DOC_BASE + 5] * 2)[0] == INVALID    # searchAfter without after values
    assert raw_sorted(gix, qs, 40, CSort(2, 0, 0, 0, 0, None), after_docs=[DOC_BASE + 5] * 2)[0] == 0   # docid needs none
    for col in (-1, len(sh.columns), 99):                                            # a bad column
        assert raw_sorted(gix, qs, 40, CSort(1, col, 0, 0, 0, None))[0] == INVALID
    assert raw_sorted(gix, qs, 40, CSort(7, 0, 0, 0, 0, None))[0] == INVALID         # a bad sort kind
    assert raw_sorted(gix, qs, 40, None)[0] == INVALID                               # no sort
    assert raw_sorted(gix, qs, 0, ok)[0] == INVALID                                  # numHits 0


# ---- the index-time codes (tests/csrc/sort_code_harness.cu) ----

def check_codes(values, has=None, int32=False):
    got, dist = sch.codes(values, has, int32)
    want, keys = sch.reference_codes(values, has)
    assert np.array_equal(got, want)
    assert np.array_equal(dist, keys)
    return dist


@pytest.mark.parametrize("int32", [False, True], ids=["int64", "int32"])
def test_codes_at_the_edges_of_shape(built, int32):
    for v, h in (([7], None), ([7], [1]), ([7], [0]), ([-3] * 1000, None), ([5] * 1000, np.arange(1000) % 2),
                 (np.arange(1000) - 500, np.zeros(1000, np.uint8))):
        dist = check_codes(v, h, int32)
        assert len(dist) == (0 if h is not None and not np.any(h) else 1 if len(set(np.asarray(v).tolist())) == 1 else len(v))
    got, dist = sch.codes(np.zeros(0, np.int64))
    assert len(got) == 0 and len(dist) == 0


def test_codes_of_the_integer_extremes(built):
    rng = np.random.default_rng(3)
    v32 = rng.integers(-1000, 1000, 50_000)
    v32[rng.choice(50_000, 40, replace=False)] = np.repeat([ss.I32_MIN, ss.I32_MAX, -1, 0], 10)
    check_codes(v32, (rng.random(50_000) < 0.8).astype(np.uint8), int32=True)
    dist = check_codes(v32, None, int32=True)
    assert dist[0] == sch.sortable([ss.I32_MIN])[0] and dist[-1] == sch.sortable([ss.I32_MAX])[0]
    v64 = rng.integers(-2**62, 2**62, 50_000, dtype=np.int64)
    v64[rng.choice(50_000, 40, replace=False)] = np.repeat(np.array([ss.I64_MIN, ss.I64_MAX, -1, 0], np.int64), 10)
    dist = check_codes(v64, None)
    assert dist[0] == sch.sortable([ss.I64_MIN])[0] and dist[-1] == sch.sortable([ss.I64_MAX])[0]


def test_codes_of_float_and_double_encodings(built):
    rng = np.random.default_rng(4)
    fspecial = np.float32([-0.0, 0.0, np.inf, -np.inf, 1e-45, -1e-45, 1e-40, -3e-39, np.finfo(np.float32).max,
                           -np.finfo(np.float32).max, np.nan])
    f = np.concatenate([fspecial, rng.normal(0, 10, 5000).astype(np.float32)])[rng.integers(0, 5011, 40_000)]
    dist = check_codes(ss._sortable_f32(f), None, int32=True)
    assert len(dist) >= len(fspecial) - 1                                   # -0 and +0 are distinct values
    dspecial = np.array([-0.0, 0.0, np.inf, -np.inf, 5e-324, -5e-324, 1e-310, np.finfo(np.float64).max,
                         -np.finfo(np.float64).max, np.nan])
    d = np.concatenate([dspecial, rng.normal(0, 1e6, 5000)])[rng.integers(0, 5010, 40_000)]
    check_codes(ss._sortable_f64(d), (rng.random(40_000) < 0.7).astype(np.uint8))


def test_codes_at_scale(built):
    rng = np.random.default_rng(5)
    v = rng.permutation(np.unique(rng.integers(-2**40, 2**40, 1_100_000)))[:1 << 20]
    assert len(np.unique(v)) == 1 << 20
    check_codes(v, None)
    check_codes(np.array([-5, 0, 2**30], np.int64)[rng.integers(0, 3, 1 << 24)], None, int32=True)


def test_code_of_every_probe_position(built):
    rng = np.random.default_rng(6)
    for held in (np.array([ss.I32_MIN, -5, -4, 0, 3, 9, ss.I32_MAX], np.int64),
                 np.unique(rng.integers(-2**62, 2**62, 3000, dtype=np.int64)),
                 np.array([ss.I64_MIN, 0, ss.I64_MAX], np.int64), np.array([42], np.int64)):
        dist = check_codes(rng.permutation(np.repeat(held, 3)))
        probes = [held, held[:-1] + 1, held[1:] - 1, held[:-1] // 2 + held[1:] // 2]   # at and between the values
        if held[0] > ss.I64_MIN:
            probes.append([held[0] - 1, ss.I64_MIN])
        if held[-1] < ss.I64_MAX:
            probes.append([held[-1] + 1, ss.I64_MAX])
        p = np.concatenate([np.asarray(x, np.int64) for x in probes])
        got = sch.code_of(dist, p)
        assert np.array_equal(got, sch.reference_code_of(dist, p))
        assert np.array_equal(got[:len(held)], 2 * np.arange(len(held)) + 2)
    assert np.array_equal(sch.code_of(np.zeros(0, np.uint64), [ss.I64_MIN, 0, ss.I64_MAX]), [1, 1, 1])


def test_harness_refuses_bad_arguments(built):
    lib = sch.lib()
    v = np.arange(4, dtype=np.int64)
    v32 = np.arange(4, dtype=np.int32)
    out, dist, nd = np.zeros(4, np.uint32), np.zeros(4, np.uint64), C.c_int32()
    assert lib.sh_codes(v.ctypes.data, v32.ctypes.data, None, 4, out.ctypes.data, dist.ctypes.data, C.byref(nd)) == sch.INVALID
    assert lib.sh_codes(None, None, None, 4, out.ctypes.data, dist.ctypes.data, C.byref(nd)) == sch.INVALID
    assert lib.sh_codes(v.ctypes.data, None, None, -1, out.ctypes.data, dist.ctypes.data, C.byref(nd)) == sch.INVALID
    bad = np.array([3, 2], np.uint64)
    assert lib.sh_code_of(bad.ctypes.data, 2, v.ctypes.data, 4, out.ctypes.data) == sch.INVALID
    assert lib.sh_code_of(dist.ctypes.data, 0, v.ctypes.data, 0, out.ctypes.data) == sch.INVALID
