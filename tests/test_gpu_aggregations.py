"""Aggregating additional collectors (terms / min / max / sum, nrtgpu_search_bool_aggs) against tests/aggs_reference.py
over the oracle's match sets, on one 1.1M-doc shard: three probe slices, heavy (query, slice) pairs split into parts,
match-all and range-led queries swept by the dense driver, every 11th doc deleted. Aggregations send every query -- pure
disjunctions too -- through the generic probe instantiation, where a doc on several SHOULD lists (or twice on the same
one) must be collected exactly once.

Columns sit where the kernels can go wrong: negatives and count ties; 1 / 2047 / 2048 / 2049 / 4097 distinct values
either side of the 2048-bucket chunk of agg_terms_topk_kernel; int64 over +-2^62 with INT64_MIN / MAX and missing
values; float and double columns with +-0, subnormals, +-inf, +-MAX, NaN and missing values; a column with no values.
Terms results, counts and MIN / MAX are exact; SUM is within n * 2^-53 * sum|v| (exact for integer columns whose
sum|v| < 2^53)."""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest

import aggs_reference as ar
import oracle
import plan_harness as ph
from nrtsearch_b200 import NrtGpuError, NrtGpuUnsupported
from nrtsearch_b200 import _native
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, GpuIndex, GpuIndexSearcher, MatchAllDocsQuery, MaxCollector,
                                   MinCollector, Occur, RangeQuery, RelevanceCollector, SumCollector, TermQuery, TermsCollector,
                                   compile_queries, double_to_sortable_long, float_to_sortable_int)

pytestmark = pytest.mark.gpu
INT_MAX = 2**31 - 1
N = 1_100_000
VOCAB = 20_000
K = 50
I64_MIN, I64_MAX = -2**63, 2**63 - 1
# columns
C_INT, D1, D2047, D2048, D2049, D4097, I64, F32, F64, NONE, SEL, UNIQ, MV = range(13)
FIELD_TYPE = {C_INT: "int", D1: "long", D2047: "long", D2048: "long", D2049: "long", D4097: "long", I64: "long",
              F32: "float", F64: "double", NONE: "long", SEL: "int", UNIQ: "long"}
# SEL marks the docs whose F32 / F64 values are NaN (1), +inf (2), -inf (3), +MAX (4), -MAX (5)
SEL_NAN, SEL_PINF, SEL_NINF, SEL_PMAX, SEL_NMAX = 1, 2, 3, 4, 5
VALUE_TYPE = {"int": ar.INT, "long": ar.INT, "float": ar.FLOAT, "double": ar.DOUBLE}


def make_columns(n, seed):
    rng = np.random.default_rng(seed)
    doc = np.arange(n, dtype=np.int64)
    cols, has = [None] * 13, [None] * 13
    cols[C_INT] = doc * 7 % 60 - 30                                  # 60 values in equal shares: count ties everywhere
    for c, d in ((D1, 1), (D2047, 2047), (D2048, 2048), (D2049, 2049), (D4097, 4097)):
        keys = np.sort(rng.choice(np.arange(-2**40, 2**40, 2**20 + 7, dtype=np.int64), d, replace=False))
        idx = (d * rng.random(n) ** 3).astype(np.int64)              # skewed counts, a long tail of small (tied) ones
        idx[rng.permutation(n)[:d]] = np.arange(d)                   # every value present: exactly d distinct
        cols[c] = keys[idx]
    pool = np.concatenate([np.array([I64_MIN, I64_MAX, 2**62, -2**62, 0, -1], np.int64),
                           rng.integers(-2**62, 2**62, 2994, dtype=np.int64)])
    cols[I64] = pool[rng.integers(0, len(pool), n)]
    cols[I64][rng.permutation(n)[:len(pool)]] = pool
    has[I64] = (rng.random(n) >= 0.3).astype(np.uint8)
    sel = np.zeros(n, np.int64)
    special = rng.permutation(n)
    for i, s in enumerate((SEL_NAN, SEL_PINF, SEL_NINF)):
        sel[special[i * 3000:(i + 1) * 3000]] = s
    sel[special[9000:9002]], sel[special[9002:9004]] = SEL_PMAX, SEL_NMAX
    cols[SEL] = sel
    f32_max = np.finfo(np.float32).max
    fpool = np.concatenate([np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, f32_max, -f32_max], np.float32),
                            rng.normal(0, 100, 2992).astype(np.float32)])
    f = fpool[rng.integers(0, len(fpool), n)]
    f[sel == SEL_NAN], f[sel == SEL_PINF], f[sel == SEL_NINF] = np.nan, np.inf, -np.inf
    f[sel == SEL_PMAX], f[sel == SEL_NMAX] = f32_max, -f32_max
    cols[F32] = np.array([float_to_sortable_int(x) for x in fpool.tolist() + [math.nan, math.inf, -math.inf]],
                         np.int64)[_index_in(f, np.concatenate([fpool, np.float32([np.nan, np.inf, -np.inf])]))]
    dpool = np.concatenate([np.array([0.0, -0.0, 5e-324, -5e-324, 1e-310, -2.5e-315, 1e300, -1e300]),
                            rng.normal(0, 1e6, 2992)])
    dv = dpool[rng.integers(0, len(dpool), n)]
    dmax = np.finfo(np.float64).max
    dv[sel == SEL_NAN], dv[sel == SEL_PINF], dv[sel == SEL_NINF] = np.nan, np.inf, -np.inf
    dv[sel == SEL_PMAX], dv[sel == SEL_NMAX] = dmax, -dmax
    b = dv.view(np.int64)
    cols[F64] = b ^ ((b >> 63) & np.int64(0x7fffffffffffffff))      # NumericUtils.doubleToSortableLong
    assert cols[F64][sel == SEL_NAN][0] == double_to_sortable_long(math.nan)
    miss = (rng.random(n) < 0.1) & (sel == 0)
    has[F32] = has[F64] = (~miss).astype(np.uint8)
    cols[NONE] = rng.integers(-5, 5, n).astype(np.int64)
    has[NONE] = np.zeros(n, np.uint8)
    cols[UNIQ] = doc * 3 - n                                        # n distinct values
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(doc % 3, out=offs[1:])                                # multi-valued: 0..2 values per doc
    owner = np.repeat(doc, doc % 3)
    cols[MV] = owner % 50 + 7 * (np.arange(int(offs[-1])) - offs[owner])   # ascending within a doc
    return cols, has, offs


def _index_in(x, pool):
    """position of every float32 in x within pool (bitwise, NaN included)"""
    kb, xb = pool.view(np.uint32), x.view(np.uint32)
    order = np.argsort(kb)
    pos = np.searchsorted(kb[order], xb)
    assert np.array_equal(kb[order][pos], xb)
    return order[pos]


@pytest.fixture(scope="module")
def setup(gpu_ctx):
    sh = ix.synth_text_shard(N, VOCAB, seed=0xA66, min_len=4, poisson_mean=10.0)
    sh.columns, sh.column_has, offs = make_columns(N, 0xA67)
    sh.column_offsets = [None] * MV + [offs]
    sh.live_docs = (np.arange(N) % 11 != 0).astype(np.uint8)
    gix = GpuIndex(gpu_ctx, sh)
    oix = oracle.OracleIndex(sh)
    yield sh, gix, oix
    gix.close()


@pytest.fixture(scope="module")
def ref(setup):
    sh, _, oix = setup
    return Reference(sh, oix, QUERIES)


def T(t):
    return TermQuery(int(t))


def bq(*clauses, msm=0):
    q = BooleanQuery()
    q.minimum_number_should_match = msm
    for c, o in clauses:
        q.add(c, o)
    return q


S, M_, F, NOT = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT

QUERIES = [
    bq((T(5), S), (T(9), S), (T(5), S)),                                  # overlapping lists, a repeated term
    bq((T(0), S), (T(1), S)),                                             # the two longest lists of the shard
    bq((T(20), S), (T(33), S), (T(50), S), (T(71), S)),
    bq((T(1500), S), (T(2300), S)),
    bq((BoostQuery(T(12), 2.5), S), (T(13), S), (T(400), S)),
    bq((T(3), M_), (T(40), M_), (RangeQuery(C_INT, -10, 10), F)),         # conjunction + range
    bq((T(12), M_), (T(100), S)),
    bq((T(8), S), (T(60), S), (T(2), NOT)),                               # MUST_NOT
    bq((T(4), S), (T(15), S), (T(30), S), (T(90), S), msm=2),             # minimumNumberShouldMatch
    MatchAllDocsQuery(),
    RangeQuery(C_INT, 0, 25),                                             # range-only: dense driver
    bq((RangeQuery(I64, 0, 2**62), F), (T(1), NOT)),
    bq((T(6), S), (RangeQuery(SEL, 1, 3), S)),                            # disjunction led by the dense driver
    bq((T(7), M_), (T(7), NOT)),                                          # has work, matches nothing
    RangeQuery(C_INT, 100, 200),                                          # matches nothing
    BooleanQuery(),                                                       # empty: no clauses
    bq((T(5), S), (T(9), S), msm=3),                                      # empty: msm > #SHOULD
    RangeQuery(SEL, SEL_NAN, SEL_NAN),                                    # only NaN
    RangeQuery(SEL, SEL_PINF, SEL_PINF),                                  # only +inf
    RangeQuery(SEL, SEL_NINF, SEL_NINF),                                  # only -inf
    RangeQuery(SEL, SEL_NAN, SEL_PINF),                                   # NaN and +inf
    RangeQuery(SEL, SEL_PMAX, SEL_NMAX),                                  # +-MAX
    bq((T(2), S), (RangeQuery(SEL, SEL_NINF, SEL_NMAX), F)),
]
EMPTY = [BooleanQuery(), bq((T(5), S), (T(9), S), msm=3)]


def terms(c, size, desc=True):
    return TermsCollector(c, size, desc, FIELD_TYPE[c])


def stat(cls, c):
    return cls(c, FIELD_TYPE[c])


# 8 aggregations per search (kMaxAggs); terms sizes 1 / 7 / 2047 / 2048 in both orders
GROUPS = [
    [terms(C_INT, 7), terms(C_INT, 7, False), terms(C_INT, 1), stat(MinCollector, C_INT), stat(MaxCollector, C_INT),
     stat(SumCollector, C_INT), terms(SEL, 7), stat(SumCollector, SEL)],
    [terms(D1, 1), terms(D2047, 2047), terms(D2048, 2048, False), terms(D2049, 2048), terms(D2049, 2047, False),
     terms(D4097, 2048), terms(D4097, 7, False), terms(D2048, 2047)],
    [terms(I64, 7), terms(I64, 2048, False), stat(MinCollector, I64), stat(MaxCollector, I64), stat(SumCollector, I64),
     terms(NONE, 3), stat(MaxCollector, NONE), stat(SumCollector, NONE)],
    [terms(F32, 7), stat(MinCollector, F32), stat(MaxCollector, F32), stat(SumCollector, F32), stat(MinCollector, F64),
     stat(MaxCollector, F64), stat(SumCollector, F64), terms(F64, 2047, False)],
    [stat(MinCollector, NONE), stat(MinCollector, D1), stat(MaxCollector, D1), stat(SumCollector, D4097), terms(F64, 7),
     terms(F32, 2048, False), terms(C_INT, 2048), terms(C_INT, 2047, False)],
]


class Reference:
    """per-query match sets and per-column value codes of one shard state (its live docs)"""

    def __init__(self, sh, oix, queries):
        carr, _, qarr, nq = compile_queries(queries)
        self.sh = sh
        self.match = [oracle.match_bitmap(oix, carr, qarr, q).astype(bool) for q in range(nq)]
        self._codes = {}

    def has(self, c):
        h = self.sh.column_has[c]
        return np.ones(self.sh.n_docs, bool) if h is None else h != 0

    def codes(self, c):
        if c not in self._codes:
            h = self.has(c)
            keys, inv = np.unique(self.sh.columns[c][h], return_inverse=True)
            code = np.full(self.sh.n_docs, -1, np.int64)
            code[h] = inv
            self._codes[c] = (keys, code)
        return self._codes[c]

    def terms(self, q, a):
        keys, code = self.codes(a.column)
        cnt = np.bincount(code[self.match[q] & (code >= 0)], minlength=len(keys))
        return ar.terms_from_counts(keys, cnt, a.size, a.order_desc)

    def values(self, q, c):
        return ar.as_doubles(self.sh.columns[c][self.match[q] & self.has(c)], VALUE_TYPE[FIELD_TYPE[c]])


def check_aggs(ref, adds, outs, rows=None):
    rows = range(len(ref.match)) if rows is None else rows
    for q in rows:
        for a, o in zip(adds, outs):
            what = f"query {q}, {type(a).__name__} column {a.column}"
            if isinstance(a, TermsCollector):
                w = ref.terms(q, a)
                assert o["n"][q] == w["n"] and o["total_buckets"][q] == w["total_buckets"], f"{what}: bucket counts"
                assert o["other_counts"][q] == w["other_counts"], f"{what}: other_counts"
                assert np.array_equal(o["keys"][q], w["keys"]) and np.array_equal(o["counts"][q], w["counts"]), f"{what} size {a.size}: buckets"
                continue
            v, got = ref.values(q, a.column), float(o[q])
            if isinstance(a, MaxCollector):
                assert got == ar.max_value(v), f"{what}: {got!r} vs {ar.max_value(v)!r}"
            elif isinstance(a, MinCollector):
                assert got == ar.min_value(v), f"{what}: {got!r} vs {ar.min_value(v)!r}"
            else:
                assert ar.sum_ok(got, v), f"{what}: {got!r} vs {ar.sum_value(v)}"
                if a.field_type in ("int", "long") and math.fsum(np.abs(v)) < 2.0**53:
                    assert got == math.fsum(v), f"{what}: integer sum not exact"


def test_plan_has_slices_parts_and_dense_items(setup):
    """The aggregation batch really is a 3-slice generic probe batch with split items (the planner on this dictionary)."""
    sh, _, _ = setup
    nd = np.array([0 if sh.column_offsets[c] is not None else len(np.unique(sh.columns[c][sh.column_has[c] != 0]))
                   if sh.column_has[c] is not None else len(np.unique(sh.columns[c])) for c in range(len(sh.columns))], np.int32)
    d = ph.Dictionary(N, sh.term_off, col_multi=np.array([c == MV for c in range(len(sh.columns))], np.uint8),
                      col_n_distinct=nd, has_deletes=True)
    aggs = [_native.Aggregation(1, C_INT, 0, 7, 1, 0)]
    p = ph.plan(d, QUERIES, K, aggs=aggs)
    try:
        assert p.n_slices == 3 and p.parts_max > 1 and p.n_probe_simple == 0 and p.n_probe_generic == p.n_work
        parts = [ph.decode(w)[2] for w in p.work_item]
        assert max(parts) > 0, "no (query, slice) pair was split"
        dense = {i for i, q in enumerate(p.queries) if q["dense_driver"]}
        assert dense and any(int(q) in dense for q in p.work_query)
        assert set(p.work_query.tolist()) == {i for i, q in enumerate(p.queries) if not q["empty"]}
        assert p.threshold == INT_MAX
    finally:
        p.close()
    assert nd[D1] == 1 and nd[D2047] == 2047 and nd[D2048] == 2048 and nd[D2049] == 2049 and nd[D4097] == 4097 and nd[NONE] == 0


@pytest.mark.parametrize("group", range(len(GROUPS)))
def test_aggregations_match_reference(setup, ref, group):
    _, gix, _ = setup
    s = GpuIndexSearcher(gix)
    adds = GROUPS[group]
    assert len(adds) == 8
    res, outs = s.search_with_collectors(QUERIES, RelevanceCollector(K, 1000), adds)
    check_aggs(ref, adds, outs)
    # the page is the one of search_batch at COMPLETE, and totalHits the match count
    plain = s.search_batch(QUERIES, RelevanceCollector(K, INT_MAX))
    assert np.array_equal(res.counts, plain.counts) and np.array_equal(res.docs, plain.docs)
    assert np.array_equal(res.scores.view(np.uint32), plain.scores.view(np.uint32))
    assert res.total_hits.tolist() == plain.total_hits.tolist() == [int(m.sum()) for m in ref.match]


def test_nan_and_infinities_never_win_min_max(setup):
    """MAX over {NaN} / {-inf} is -Double.MAX_VALUE, MIN over {NaN} / {+inf} is Double.MAX_VALUE (MaxCollectorManager:117)."""
    sh, gix, oix = setup
    qs = [RangeQuery(SEL, SEL_NAN, SEL_NAN), RangeQuery(SEL, SEL_PINF, SEL_PINF), RangeQuery(SEL, SEL_NINF, SEL_NINF),
          RangeQuery(SEL, SEL_NAN, SEL_PINF),
          bq((T(0), S), (RangeQuery(SEL, SEL_NAN, SEL_NAN), S), (RangeQuery(SEL, SEL_PINF, SEL_PINF), NOT))]
    adds = [stat(MaxCollector, F32), stat(MinCollector, F32), stat(MaxCollector, F64), stat(MinCollector, F64)]
    _, outs = GpuIndexSearcher(gix).search_with_collectors(qs, RelevanceCollector(10, INT_MAX), adds)
    D, f32_max = ar.DBL_MAX, float(np.finfo(np.float32).max)
    assert outs[0][:4].tolist() == [-D, math.inf, -D, math.inf] and outs[1][:4].tolist() == [D, D, -math.inf, D]
    assert outs[2][:4].tolist() == [-D, math.inf, -D, math.inf] and outs[3][:4].tolist() == [D, D, -math.inf, D]
    assert not np.isnan(outs[0][4]) and outs[0][4] == f32_max    # NaN docs among ordinary ones: the ordinary max wins
    check_aggs(Reference(sh, oix, qs), adds, outs)


def test_repeated_call_is_identical(setup):
    _, gix, _ = setup
    s = GpuIndexSearcher(gix)
    adds = GROUPS[0][:6] + [stat(MinCollector, F64), stat(MaxCollector, F32)]
    r1, o1 = s.search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX), adds)
    r2, o2 = s.search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX), adds)
    assert np.array_equal(r1.docs, r2.docs) and np.array_equal(r1.total_hits, r2.total_hits)
    for a, x, y in zip(adds, o1, o2):
        if isinstance(a, TermsCollector):
            assert all(np.array_equal(x[k], y[k]) for k in x)
        else:
            assert np.array_equal(x.view(np.int64), y.view(np.int64))


def test_aggregations_follow_live_docs_updates(setup):
    sh, gix, _ = setup
    s = GpuIndexSearcher(gix)
    adds = [terms(C_INT, 7), terms(D2049, 2048), stat(MinCollector, I64), stat(MaxCollector, F64), stat(SumCollector, C_INT),
            stat(SumCollector, F32)]
    qs = QUERIES[:13]
    more = ((np.arange(N) % 11 != 0) & (np.arange(N) % 7 != 3)).astype(np.uint8)
    try:
        for live in (more, None):
            gix.set_live_docs(live)
            sh2 = dataclasses.replace(sh, live_docs=live)
            _, outs = s.search_with_collectors(qs, RelevanceCollector(K, INT_MAX), adds)
            check_aggs(Reference(sh2, oracle.OracleIndex(sh2), qs), adds, outs)
    finally:
        gix.set_live_docs(sh.live_docs)


EMPTY_ADDS = [stat(MinCollector, C_INT), stat(MaxCollector, F64), stat(SumCollector, I64)]


def check_unset(res, outs, adds):
    D = ar.DBL_MAX
    assert not res.counts.any() and not res.total_hits.any()
    for a, o in zip(adds, outs):
        if isinstance(a, TermsCollector):
            assert not o["n"].any() and not o["total_buckets"].any() and not o["other_counts"].any()
            assert not o["keys"].any() and not o["counts"].any()
        else:
            want = D if isinstance(a, MinCollector) else -D if isinstance(a, MaxCollector) else 0.0
            assert o.tolist() == [want] * len(o), f"{type(a).__name__}: {o.tolist()}"


def test_all_empty_batch_after_a_larger_call_on_the_same_index(setup):
    """A batch without work items must not return what the pooled workspace holds from an earlier call."""
    _, gix, _ = setup
    s = GpuIndexSearcher(gix)
    _, outs = s.search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX), EMPTY_ADDS)
    assert outs[0][0] != ar.DBL_MAX and outs[2][0] != 0.0
    res, outs = s.search_with_collectors(EMPTY, RelevanceCollector(K, INT_MAX), EMPTY_ADDS)
    check_unset(res, outs, EMPTY_ADDS)
    adds = [terms(C_INT, 7)] + EMPTY_ADDS
    s.search_with_collectors(QUERIES, RelevanceCollector(K, INT_MAX), adds)
    res, outs = s.search_with_collectors(EMPTY, RelevanceCollector(K, INT_MAX), adds)
    check_unset(res, outs, adds)


def test_all_empty_batch_on_a_fresh_index(gpu_ctx):
    n = 60_000
    sh = ix.synth_text_shard(n, 2_000, seed=0xA68, min_len=4, poisson_mean=10.0)
    sh.columns, sh.column_has, offs = make_columns(n, 0xA69)
    sh.column_offsets = [None] * MV + [offs]
    gix = GpuIndex(gpu_ctx, sh)
    try:
        adds = [terms(C_INT, 7), terms(NONE, 2)] + EMPTY_ADDS
        res, outs = GpuIndexSearcher(gix).search_with_collectors(EMPTY, RelevanceCollector(5, INT_MAX), adds)
        check_unset(res, outs, adds)
    finally:
        gix.close()


def raw_search_aggs(gix, queries, k, aggs):
    """nrtgpu_search_bool_aggs with hand-made aggregation records (what the collector classes cannot express)"""
    lib = _native.gpu_lib()
    carr, ncl, qarr, nq = compile_queries(queries)
    arr = (_native.Aggregation * len(aggs))(*aggs)
    bufs = [np.zeros(nq * max(a.size, 1), np.int64) for a in aggs]
    res = (_native.AggregationResult * len(aggs))(*[_native.AggregationResult(b.ctypes.data, None, None, None, None, None) for b in bufs])
    docs, scores, counts, total = np.zeros((nq, k), np.int32), np.zeros((nq, k), np.float32), np.zeros(nq, np.int32), np.zeros(nq, np.int64)
    _native.check(lib.nrtgpu_search_bool_aggs(gix.handle, carr, ncl, qarr, nq, k, 0, arr, len(aggs), res, C.c_void_p(0),
                                              docs.ctypes.data, scores.ctypes.data, counts.ctypes.data, total.ctypes.data))


def test_refusals(setup):
    sh, gix, _ = setup
    s = GpuIndexSearcher(gix)
    qs = QUERIES[:3]
    A = _native.Aggregation

    def refused(exc, status, msg, fn):
        with pytest.raises(exc) as e:
            fn()
        assert e.value.status == status and msg in e.value.message, e.value.message

    refused(NrtGpuError, 1, "at most 8 aggregations per search",
            lambda: s.search_with_collectors(qs, RelevanceCollector(K), [stat(MinCollector, C_INT)] * 9))
    for size in (0, 2049):
        refused(NrtGpuUnsupported, 3, "size must be in [1, 2048]",
                lambda: s.search_with_collectors(qs, RelevanceCollector(K), [terms(C_INT, size)]))
    refused(NrtGpuUnsupported, 3, "aggregation on a multi-valued column",
            lambda: s.search_with_collectors(qs, RelevanceCollector(K), [MinCollector(MV)]))
    for kind in (0, 5):
        refused(NrtGpuError, 1, "bad aggregation kind", lambda: raw_search_aggs(gix, qs, K, [A(kind, C_INT, 0, 1, 1, 0)]))
    for col in (-1, len(sh.columns)):
        refused(NrtGpuError, 1, "aggregation column out of range", lambda: raw_search_aggs(gix, qs, K, [A(2, col, 0, 0, 0, 0)]))
    for vt in (-1, 3):
        refused(NrtGpuError, 1, "bad aggregation value_type", lambda: raw_search_aggs(gix, qs, K, [A(3, C_INT, vt, 0, 0, 0)]))
    five = bq(*[(T(t), S) for t in (5, 9, 20, 33, 50)])
    refused(NrtGpuUnsupported, 3, "more than 4 term clauses or top_k > 512",
            lambda: s.search_with_collectors([five], RelevanceCollector(K), [stat(SumCollector, C_INT)]))
    refused(NrtGpuUnsupported, 3, "more than 4 term clauses or top_k > 512",
            lambda: s.search_with_collectors(qs, RelevanceCollector(513), [stat(SumCollector, C_INT)]))
    # the count table of a terms aggregation: nq x distinct values x 4 bytes; just over 2 GB is refused before any allocation
    nq = (2**29) // (N - N // 11) + 1   # (whether or not deleted docs' values are counted)
    refused(NrtGpuUnsupported, 3, "exceeds the 2 GB count table",
            lambda: s.search_with_collectors([MatchAllDocsQuery()] * nq, RelevanceCollector(1), [terms(UNIQ, 1)]))
    # the index still answers afterwards
    _, outs = s.search_with_collectors(qs, RelevanceCollector(K), [stat(MaxCollector, C_INT)])
    assert outs[0].tolist() == [29.0] * 3
