"""Shards, queries, Sorts and after FieldDocs for the one-field sorted search (nrtgpu_search_sorted), shared by its GPU
tests (tests/test_gpu_sort_single.py) and the CPU test that pins its two references to each other
(tests/test_sort_single_reference.py). Columns are built in numpy where the value codes can go wrong: int32 with
negatives and INT32_MIN / MAX held (the missing value is held: exact ties between holders and docs without a value),
int32 without a has mask, int64 over +-2^62 without Long.MIN / MAX (odd missing code at both ends), float and double with
-0, +0, subnormals, +-MAX and NaN (+inf held by the float column only, -inf by neither), one distinct value, no value at
all. A 3,000-doc group ties on one value in every sortable column (placed across a probe slice edge by the GPU tests).

The two references: oracle.search_sorted (the C oracle's TopFieldCollector) and the one-field Sorts of
sort_fields_reference.search_sorted_fields (a numpy lexsort over the oracle's matches)."""
from __future__ import annotations

import numpy as np

import oracle
import sort_fields_reference as ref
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (BooleanQuery, FieldDoc, MatchAllDocsQuery, Occur, RangeQuery, ScoreDoc, SortType, TermQuery,
                                   compile_queries, double_to_sortable_long, float_to_sortable_int)

I32_MIN, I32_MAX, I64_MIN, I64_MAX = -2**31, 2**31 - 1, -2**63, 2**63 - 1
TIE_DOCS = 3000
VOCAB = 20_000
# columns
C_I32, C_I32_FULL, C_I64, C_F32, C_F64, C_ONE, C_NONE, C_TAG, C_KEY, C_MV = range(10)
FIELD_TYPE = {C_I32: "int", C_I32_FULL: "int", C_I64: "long", C_F32: "float", C_F64: "double", C_ONE: "int", C_NONE: "long"}
SORT_COLUMNS = list(FIELD_TYPE)
TIE_VALUE = {C_I32: 17, C_I32_FULL: 0, C_I64: 2**61, C_F32: float_to_sortable_int(1.5), C_F64: double_to_sortable_long(2.5),
             C_ONE: 42}
EXACT_K = 40                  # C_KEY == 1 on exactly EXACT_K live docs, == 2 on EXACT_K - 1


def _sortable_f32(f):
    b = np.asarray(f, np.float32).view(np.int32).astype(np.int64)
    return b ^ ((b >> 31) & 0x7fffffff)                                # NumericUtils.floatToSortableInt


def _sortable_f64(d):
    b = np.asarray(d, np.float64).view(np.int64)
    return b ^ ((b >> 63) & np.int64(0x7fffffffffffffff))              # NumericUtils.doubleToSortableLong


def make_columns(n, live, tie_lo, seed=0x5017):
    """(columns, has masks, offsets of the multi-valued column); live = the live docs, tie_lo = the tie group's first doc"""
    rng = np.random.default_rng(seed)
    tie = np.zeros(n, bool)
    tie[tie_lo:tie_lo + TIE_DOCS] = True
    base_miss = (rng.random(n) < 0.2) & ~tie                           # docs without a value in every sparse column
    cols, has = [None] * 10, [None] * 10
    c = rng.integers(-5000, 5000, n).astype(np.int64)
    for v in (I32_MIN, I32_MAX):                                        # held by a few docs: the missing value is held
        c[rng.choice(np.nonzero(~base_miss & ~tie)[0], 4, replace=False)] = v
    cols[C_I32], has[C_I32] = c, ~base_miss
    cols[C_I32_FULL] = rng.integers(-3000, 3000, n).astype(np.int64) * 700_001
    pool = np.concatenate([np.array([2**62, -2**62, 0, -1, 2**61], np.int64), rng.integers(-2**62, 2**62, 4995, dtype=np.int64)])
    cols[C_I64] = pool[rng.integers(0, len(pool), n)]
    has[C_I64] = ~(base_miss | ((rng.random(n) < 0.07) & ~tie))
    f32_max = np.finfo(np.float32).max
    fpool = np.concatenate([np.float32([0.0, -0.0, np.inf, np.nan, 1e-45, -1e-45, 1e-40, -3e-39, f32_max, -f32_max]),
                            rng.normal(0, 100, 2990).astype(np.float32)])
    cols[C_F32] = _sortable_f32(fpool[rng.integers(0, len(fpool), n)])
    has[C_F32] = ~(base_miss | ((rng.random(n) < 0.12) & ~tie))
    dmax = np.finfo(np.float64).max
    dpool = np.concatenate([np.array([0.0, -0.0, np.nan, 5e-324, -5e-324, 1e-310, -2.5e-315, dmax, -dmax]), rng.normal(0, 1e6, 2991)])
    cols[C_F64] = _sortable_f64(dpool[rng.integers(0, len(dpool), n)])
    has[C_F64] = ~(base_miss | ((rng.random(n) < 0.1) & ~tie))
    cols[C_ONE], has[C_ONE] = np.full(n, 42, np.int64), ~base_miss
    cols[C_NONE], has[C_NONE] = rng.integers(-9, 9, n).astype(np.int64), np.zeros(n, bool)
    for col, v in TIE_VALUE.items():
        cols[col][tie] = v
    cols[C_TAG] = base_miss.astype(np.int64)                            # RangeQuery(C_TAG, 1, 1): only docs without a value
    key = np.zeros(n, np.int64)
    pick = rng.choice(np.nonzero(live)[0], 2 * EXACT_K - 1, replace=False)
    key[pick[:EXACT_K]], key[pick[EXACT_K:]] = 1, 2
    cols[C_KEY] = key
    cnt = np.arange(n) % 3                                              # multi-valued: 0..2 values per doc
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(cnt, out=offs[1:])
    owner = np.repeat(np.arange(n), cnt)
    cols[C_MV] = owner % 50 + 7 * (np.arange(int(offs[-1])) - offs[owner])   # ascending within a doc
    has = [None if h is None else np.ascontiguousarray(h, np.uint8) for h in has]
    return cols, has, offs


def make_shard(n, doc_base, tie_lo, vocab=VOCAB, seed=0x5017):
    """n docs at doc_base, 8 % deleted, the tie group at local docs [tie_lo, tie_lo + 3000)"""
    sh = ix.synth_text_shard(n, vocab, seed=seed, min_len=4, poisson_mean=10.0)
    sh.doc_base = doc_base
    live = np.random.default_rng(seed + 1).random(n) >= 0.08
    sh.columns, sh.column_has, offs = make_columns(n, live, tie_lo, seed)
    sh.column_offsets = [None] * C_MV + [offs]
    sh.live_docs = live.astype(np.uint8)
    return sh


def T(t):
    return TermQuery(int(t))


def bq(*clauses):
    q = BooleanQuery()
    for c, o in clauses:
        q.add(c, o)
    return q


S, M_, F, NOT = Occur.SHOULD, Occur.MUST, Occur.FILTER, Occur.MUST_NOT
QUERIES = [
    bq((T(40), S), (T(300), S), (T(2000), S)),                           # pure disjunction
    bq((T(3), M_), (T(25), M_), (RangeQuery(C_I32, -2000, 2000), F)),   # conjunction + FILTER range
    bq((T(8), S), (T(60), S), (T(2), NOT)),                              # MUST_NOT
    MatchAllDocsQuery(),
    RangeQuery(C_I32, -60, 60),                                          # range-led: the dense driver, the tie group
    BooleanQuery(),                                                      # empty
    bq((T(100), M_), (RangeQuery(C_TAG, 1, 1), F)),                      # only docs without a value
    RangeQuery(C_KEY, 1, 1),                                             # exactly EXACT_K matches
    RangeQuery(C_KEY, 2, 2),                                             # EXACT_K - 1 matches
    bq((T(3000), S), (RangeQuery(C_I32, 17, 18), S)),                    # the tie group and a few hundred more
]
MATCH_ALL, EMPTY, ONLY_MISSING = 3, 5, 6


def sorts():
    """each sortable column ascending / descending, missing first / last, then docid ascending / descending"""
    out = [SortType(c, rev, last, FIELD_TYPE[c]) for c in SORT_COLUMNS for rev in (False, True) for last in (False, True)]
    return out + [SortType("docid", False), SortType("docid", True)]


def sort_id(st) -> str:
    if st.field == "docid":
        return "docid-" + ("desc" if st.reverse else "asc")
    return f"c{st.field}{FIELD_TYPE[st.field]}-{'desc' if st.reverse else 'asc'}-{'last' if st.missing_last else 'first'}"


def fields_of(st):
    return [(2, 0, int(st.reverse), 0, 0)] if st.field == "docid" else [(1, int(st.field), int(st.reverse), 0, st.missing_value())]


def _compiled(qs, after):
    sd = None if after is None else [None if a is None else ScoreDoc(a.doc, 0.0) for a in after]
    av = None if after is None else [0 if a is None else a.value for a in after]
    return compile_queries(qs, sd), av


def want_oracle(sh, qs, k, st, after=None, oix=None):
    """oracle.search_sorted: docs [nq, k] (global), values [nq, k], counts, exact totals"""
    (carr, ncl, qarr, nq), av = _compiled(qs, after)
    docid = st.field == "docid"
    return oracle.search_sorted(oix or oracle.OracleIndex(sh), carr, ncl, qarr, nq, k, 2 if docid else 1, 0 if docid else st.field,
                                st.reverse, 0 if docid else st.missing_value(), av)


def want_fields(sh, qs, k, st, after=None, oix=None):
    """the one-field Sort through sort_fields_reference.search_sorted_fields, in the shape of want_oracle"""
    (carr, ncl, qarr, nq), av = _compiled(qs, after)
    d, v, c, t = ref.search_sorted_fields(sh, carr, ncl, qarr, nq, k, fields_of(st), None if av is None else [[a] for a in av], oix)
    return d, v[:, :, 0], c, t


def after_values(sh, col, missing):
    """(name, value) after values of one column: below its minimum, between two held values, above its maximum, the
    Sort's missing value, INT32_MIN when held"""
    h = sh.column_has[col]
    held = np.unique(sh.columns[col] if h is None else sh.columns[col][h != 0])
    out = [("missing", missing)]
    if not len(held):
        return out + [("any", 0)]
    gap = np.nonzero(np.diff(held) > 1)[0]
    if held[0] > I64_MIN:
        out.append(("below", int(held[0]) - 1))
    if len(gap):
        out.append(("between", int(held[gap[len(gap) // 2]]) + 1))
    if held[-1] < I64_MAX:
        out.append(("above", int(held[-1]) + 1))
    if held[0] == I32_MIN:
        out.append(("int32-min", I32_MIN))
    if FIELD_TYPE[col] == "int":   # an int field's FieldDoc holds an Integer
        out = [(n, v) for n, v in out if I32_MIN <= v <= I32_MAX]
    return out


def synthetic_afters(sh, st, queries, after_docs):
    """(query list, FieldDoc list): every query with every after value of the Sort's column and every after doc"""
    vals = [("doc", None)] if st.field == "docid" else after_values(sh, st.field, st.missing_value())
    qs, after = [], []
    for q in queries:
        for _, v in vals:
            for d in after_docs:
                qs.append(q)
                after.append(FieldDoc(int(d), int(d if v is None else v)))   # a doc id Sort's FieldDoc holds the doc
    return qs, after


def merge_pages(st, pages, k):
    """TopFieldCollector's merge of leaf pages [(docs, values, count)] by (value in sort order, global doc): (docs, values)"""
    docs = np.concatenate([p[0][:p[2]] for p in pages]).astype(np.int64)
    vals = np.concatenate([p[1][:p[2]] for p in pages]).astype(np.int64)
    key = ref.field_keys(fields_of(st)[0], vals)
    order = np.lexsort((docs, key))[:k]
    return docs[order], vals[order]
