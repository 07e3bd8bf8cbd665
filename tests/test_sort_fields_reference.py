"""The reference for sorts of several fields (tests/sort_fields_reference.py), the checker of the multi-field sorted search
(tests/test_gpu_sort_fields.py), pinned on the CPU:
against the reference's own known answers (SortFieldTest.java:69-605: single int / long / float / double fields and their
multi-valued twins under the MIN and MAX selectors, ten segments of ten docs), and against an independent Python restatement
of TopFieldCollector's comparator on a random index with ties, missing values, a multi-valued column, deletes, a leading
score and searchAfter tuples."""
import numpy as np
import pytest

import oracle
import sort_fields_reference as ref
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import (MatchAllDocsQuery, BooleanQuery, Occur, RangeQuery, ScoreDoc, TermQuery, compile_queries,
                                   double_to_sortable_long, float_to_sortable_int)

COLUMN, DOCID, SCORE = 1, 2, 3
N_DOCS, SEG = 100, 10


def kat_segment(s):
    """docs 10*s .. 10*s+9 of SortFieldTest.initTestIndex: one segment of the 100-doc index"""
    i = np.arange(s * SEG, (s + 1) * SEG)
    iv = (i + 10) % N_DOCS - 10
    lv = ((i + 66) % N_DOCS) * 2 - 10
    fv = (((i + 33) % N_DOCS).astype(np.float32) * np.float32(1.25) - np.float32(10.0)).astype(np.float32)
    dv = ((i + 90) % N_DOCS) * 2.75 - 10.0
    fs = [float_to_sortable_int(x) for x in fv]
    fs2 = [float_to_sortable_int(x) for x in fv + np.float32(2.0)]
    ds = [double_to_sortable_long(x) for x in dv]
    ds2 = [double_to_sortable_long(x) for x in dv + 2.0]
    off = np.arange(0, 2 * SEG + 1, 2, dtype=np.int64)
    single = [iv, lv, fs, ds]
    multi = [np.stack([iv, iv + 2], 1), np.stack([lv, lv + 2], 1), np.stack([fs, fs2], 1), np.stack([ds, ds2], 1)]
    sh = ix.HostShard(SEG, s * SEG, np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros(0, np.int32),
                      [ix.TextField(None, SEG, SEG)])
    sh.columns = [np.asarray(c, np.int64) for c in single] + [np.asarray(m, np.int64).reshape(-1) for m in multi]
    sh.column_has = [None] * 8
    sh.column_offsets = [None] * 4 + [off] * 4
    return sh


def kat_top5(column, reverse=False, selector=0):
    """top 5 of a match-all query over the ten segments, each searched on its own and merged by (value, doc)"""
    carr, ncl, qarr, nq = compile_queries([MatchAllDocsQuery()])
    hits = []
    for s in range(N_DOCS // SEG):
        d, v, c, t = ref.search_sorted_fields(kat_segment(s), carr, ncl, qarr, nq, 5,
                                                 [(COLUMN, column, int(reverse), selector, -(2**63))])
        assert t[0] == SEG
        hits += [(int(v[0, r, 0]), int(d[0, r])) for r in range(c[0])]
    hits.sort(key=lambda h: (-h[0] if reverse else h[0], h[1]))
    return [h[1] for h in hits[:5]], [h[0] for h in hits[:5]]


F = float_to_sortable_int
D = double_to_sortable_long
KAT = [  # (column, reverse, selector, ids, values): SortFieldTest.java, the multi_* fields hold v and v + 2
    (0, False, 0, range(90, 95), [-10, -9, -8, -7, -6]),                        # testSortIntField
    (4, False, 0, range(90, 95), [-10, -9, -8, -7, -6]),                        # testSortMultiIntField (:188-217)
    (4, False, 1, range(90, 95), [-8, -7, -6, -5, -4]),                         # testSortMultiIntField_max (:220-249)
    (0, True, 0, range(89, 84, -1), [89, 88, 87, 86, 85]),                      # testReverseSortIntField
    (4, True, 0, range(89, 84, -1), [89, 88, 87, 86, 85]),                      # testReverseSortMultiIntField (:257-287)
    (1, False, 0, range(34, 39), [-10, -8, -6, -4, -2]),                        # testSortLongField
    (5, False, 0, range(34, 39), [-10, -8, -6, -4, -2]),                        # testSortMultiLongField
    (5, False, 1, range(34, 39), [-8, -6, -4, -2, 0]),                          # testSortMultiLongField_max
    (1, True, 0, range(33, 28, -1), [188, 186, 184, 182, 180]),                 # testReverseSortLongField
    (5, True, 0, range(33, 28, -1), [188, 186, 184, 182, 180]),                 # testReverseSortMultiLongField
    (2, False, 0, range(67, 72), [F(x) for x in (-10.0, -8.75, -7.5, -6.25, -5.0)]),      # testSortFloatField
    (6, False, 0, range(67, 72), [F(x) for x in (-10.0, -8.75, -7.5, -6.25, -5.0)]),      # testSortMultiFloatField
    (6, False, 1, range(67, 72), [F(x) for x in (-8.0, -6.75, -5.5, -4.25, -3.0)]),       # testSortMultiFloatField_max
    (2, True, 0, range(66, 61, -1), [F(x) for x in (113.75, 112.5, 111.25, 110.0, 108.75)]),   # testReverseSortFloatField
    (6, True, 0, range(66, 61, -1), [F(x) for x in (113.75, 112.5, 111.25, 110.0, 108.75)]),   # ...MultiFloatField
    (3, False, 0, range(10, 15), [D(x) for x in (-10.0, -7.25, -4.5, -1.75, 1.0)]),       # testSortDoubleField
    (7, False, 0, range(10, 15), [D(x) for x in (-10.0, -7.25, -4.5, -1.75, 1.0)]),       # testSortMultiDoubleField
    (7, False, 1, range(10, 15), [D(x) for x in (-8.0, -5.25, -2.5, 0.25, 3.0)]),         # testSortMultiDoubleField_max
    (3, True, 0, range(9, 4, -1), [D(x) for x in (262.25, 259.5, 256.75, 254.0, 251.25)]),   # testReverseSortDoubleField
    (7, True, 0, range(9, 4, -1), [D(x) for x in (262.25, 259.5, 256.75, 254.0, 251.25)]),   # ...MultiDoubleField
]


@pytest.mark.parametrize("column,reverse,selector,ids,values", KAT)
def test_sort_field_test_known_answers(column, reverse, selector, ids, values):
    got_ids, got_values = kat_top5(column, reverse, selector)
    assert got_ids == list(ids)
    assert got_values == list(values)


# ---- independent restatement: Python tuples over the matching docs ----

def random_shard(n=12_000, vocab=600, seed=17):
    sh = ix.synth_text_shard(n, vocab, min_len=4, poisson_mean=10.0)
    sh.doc_base = 5_000
    rng = np.random.default_rng(seed)
    low = rng.integers(0, 6, n).astype(np.int64)                    # heavy ties
    has_low = (rng.random(n) > 0.15).astype(np.uint8)
    big = rng.integers(-3, 3, n).astype(np.int64) * (2**61)          # long values, extremes of the domain nearby
    has_big = (rng.random(n) > 0.3).astype(np.uint8)
    cnt = rng.integers(0, 4, n)
    off = np.zeros(n + 1, np.int64)
    np.cumsum(cnt, out=off[1:])
    mv = np.sort(rng.integers(-5, 5, (n, 3)), axis=1)
    vals = np.concatenate([mv[d, :cnt[d]] for d in range(n)]).astype(np.int64)
    sh.columns = [low, big, vals]
    sh.column_has = [has_low, has_big, None]
    sh.column_offsets = [None, None, off]
    sh.live_docs = (rng.random(n) > 0.1).astype(np.uint8)
    return sh


def doc_value(sh, f, d, score):
    kind, col, _, sel, missing = f
    if kind == DOCID:
        return d + sh.doc_base
    if kind == SCORE:
        return int(np.float32(score).view(np.uint32))
    if sh.column_offsets[col] is not None:
        a, b = sh.column_offsets[col][d], sh.column_offsets[col][d + 1]
        return missing if a == b else int(sh.columns[col][b - 1 if sel == 1 else a])
    h = sh.column_has[col]
    return missing if (h is not None and not h[d]) else int(sh.columns[col][d])


def tuple_key(fields, values):
    """ascending comparator key of a FieldDoc: fields after a doc id do not count"""
    key = []
    for f, v in zip(fields, values):
        if f[0] == SCORE:
            s = float(np.uint32(v).view(np.float32))
            key.append(s if f[2] else -s)
        else:
            key.append(-v if f[2] else v)
        if f[0] == DOCID:
            break
    return tuple(key)


def expected(sh, oix, carr, qarr, q, fields, k, after=None):
    m = np.nonzero(oracle.match_bitmap(oix, carr, qarr, q))[0]
    sc = np.zeros((1, 0), np.float32)
    if len(m):
        one = (type(qarr[q]) * 1)(qarr[q])
        _, sc = oracle.score_docs(oix, carr, one, 1, (m + sh.doc_base)[None, :].astype(np.int32))
    rows =[(tuple_key(fields, vals), int(d) + sh.doc_base, vals)
            for d, s in zip(m, sc[0]) for vals in [tuple(doc_value(sh, f, int(d), s) for f in fields)]]
    if after is not None:
        avals, adoc = after
        ak = tuple_key(fields, avals)
        rows = [r for r in rows if (r[0], r[1]) > (ak, adoc)]
    rows.sort(key=lambda r: (r[0], r[1]))
    return len(m), [r[1] for r in rows[:k]], [list(r[2]) for r in rows[:k]]


SPECS = [
    [(COLUMN, 0, 0, 0, -(2**63)), (COLUMN, 1, 1, 0, 2**63 - 1)],
    [(COLUMN, 2, 0, 0, 2**63 - 1), (COLUMN, 0, 1, 0, -(2**63))],
    [(COLUMN, 2, 1, 1, -(2**63))],
    [(COLUMN, 0, 0, 0, 3), (DOCID, 0, 1, 0, 0), (COLUMN, 1, 0, 0, 0)],
    [(SCORE, 0, 0, 0, 0)],
    [(SCORE, 0, 1, 0, 0), (COLUMN, 0, 1, 0, -(2**63))],
    [(SCORE, 0, 0, 0, 0), (COLUMN, 2, 0, 1, -(2**63)), (COLUMN, 1, 0, 0, 2**63 - 1)],
]


def queries(vocab, n=10, seed=4):
    terms = ix.synth_query_terms(n, 2, vocab, seed=seed, log10_lo=0.3, log10_hi=3.0)
    qs = []
    for i, t in enumerate(terms):
        if i % 4 == 0:
            qs.append(BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD).add(TermQuery(int(t[1])), Occur.SHOULD))
        elif i % 4 == 1:
            qs.append(BooleanQuery().add(TermQuery(int(t[0])), Occur.MUST).add(RangeQuery(0, 1, 4), Occur.FILTER))
        elif i % 4 == 2:
            qs.append(MatchAllDocsQuery())
        else:
            qs.append(BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD).add(TermQuery(int(t[1])), Occur.MUST_NOT)
                      .add(RangeQuery(2, -2, 2), Occur.SHOULD))
    return qs


@pytest.mark.parametrize("spec", range(len(SPECS)))
def test_sort_fields_match_a_python_restatement(spec):
    sh = random_shard()
    oix = oracle.OracleIndex(sh)
    fields = SPECS[spec]
    qs = queries(600)
    carr, ncl, qarr, nq = compile_queries(qs)
    k = 30
    d, v, c, t = ref.search_sorted_fields(sh, carr, ncl, qarr, nq, k, fields)
    for q in range(nq):
        total, wd, wv = expected(sh, oix, carr, qarr, q, fields, k)
        assert t[q] == total and c[q] == len(wd)
        assert list(d[q, :c[q]]) == wd, (spec, q)
        assert v[q, :c[q]].tolist() == wv, (spec, q)
    # searchAfter: after tuples of page 1, and tuples of values no doc holds, with after_doc below / inside / above the leaf
    rng = np.random.default_rng(spec)
    after = []
    for q in range(nq):
        if q % 3 == 0 and c[q] > 10:
            after.append((tuple(int(x) for x in v[q, 9]), int(d[q, 9])))
        else:
            vals = []
            for f in fields:
                if f[0] == SCORE:
                    vals.append(int(np.float32(rng.random() * 4).view(np.uint32)))
                elif f[0] == DOCID:
                    vals.append(int(rng.integers(0, sh.doc_base + sh.n_docs + 100)))
                else:
                    vals.append(int(rng.integers(-3, 3)) * (2**61 if f[1] == 1 else 2) + (1 if q % 3 == 2 else 0))
            after.append((tuple(vals), int(rng.choice([0, sh.doc_base + sh.n_docs // 2, sh.doc_base + sh.n_docs + 7]))))
    sd = [ScoreDoc(a[1], 0.0) for a in after]
    carr2, ncl2, qarr2, nq2 = compile_queries(qs, sd)
    d2, v2, c2, t2 = ref.search_sorted_fields(sh, carr2, ncl2, qarr2, nq2, k, fields, [a[0] for a in after])
    for q in range(nq):
        total, wd, wv = expected(sh, oix, carr2, qarr2, q, fields, k, after[q])
        assert t2[q] == total
        assert list(d2[q, :c2[q]]) == wd, (spec, q, after[q])
        assert v2[q, :c2[q]].tolist() == wv
        if q % 3 == 0 and c[q] == k:   # page 2 continues page 1 without gap or overlap
            assert list(d2[q, :k - 10]) == list(d[q, 10:])


def test_score_first_agrees_with_the_relevance_search():
    sh = random_shard()
    oix = oracle.OracleIndex(sh)
    qs = queries(600)
    carr, ncl, qarr, nq = compile_queries(qs)
    d, v, c, t = ref.search_sorted_fields(sh, carr, ncl, qarr, nq, 20, [(SCORE, 0, 0, 0, 0)])
    wd, ws, wc, wt, _ = oracle.search_compiled(oix, carr, ncl, qarr, nq, 20)
    assert np.array_equal(c, wc) and np.array_equal(t, wt)
    for q in range(nq):
        assert np.array_equal(d[q, :c[q]], wd[q, :c[q]])
        assert np.array_equal(v[q, :c[q], 0].astype(np.uint32), ws[q, :c[q]].view(np.uint32))


def test_bad_specs_are_refused():
    sh = kat_segment(0)
    oix = oracle.OracleIndex(sh)
    carr, ncl, qarr, nq = compile_queries([MatchAllDocsQuery()])
    for fields in ([], [(COLUMN, 8, 0, 0, 0)], [(COLUMN, 0, 0, 2, 0)], [(4, 0, 0, 0, 0)], [(COLUMN, 0, 0, 0, 0), (SCORE, 0, 0, 0, 0)],
                   [(DOCID, 0, 0, 0, 0)] * 9):
        with pytest.raises(ValueError):
            ref.search_sorted_fields(sh, carr, ncl, qarr, nq, 5, fields)
