"""The two references of the one-field sorted search (tests/test_gpu_sort_single.py), pinned to each other and to hand-made
answers on the CPU: oracle.search_sorted (the C oracle's TopFieldCollector) equals the one-field Sorts of
sort_fields_reference.search_sorted_fields for every Sort, page walk and after FieldDoc of the GPU module, on the same
shard builder at a smaller size; and on 20-doc leaves, an after FieldDoc that carries the missing value ties with the docs
without a value whether or not any doc holds that value, so the missing docs above after_doc come first."""
import numpy as np
import pytest

import oracle
import sort_single_shard as ss
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import FieldDoc, MatchAllDocsQuery, SortType, compile_queries, float_to_sortable_int

N, DOC_BASE, TIE_LO = 120_000, 5_000, 58_500
K_WALK, WALK_PAGES = 97, 12
SORTS = ss.sorts()


@pytest.fixture(scope="module")
def shard():
    sh = ss.make_shard(N, DOC_BASE, TIE_LO, vocab=4_000)
    return sh, oracle.OracleIndex(sh)


def assert_same(a, b, what):
    wd, wv, wc, wt = a
    gd, gv, gc, gt = b
    assert np.array_equal(wc, gc) and np.array_equal(wt, gt), what
    for q in range(len(wc)):
        assert np.array_equal(wd[q, :wc[q]], gd[q, :gc[q]]), (what, q)
        assert np.array_equal(wv[q, :wc[q]], gv[q, :gc[q]]), (what, q)


def test_queries_reach_their_edges(shard):
    sh, oix = shard
    _, _, c, t = ss.want_oracle(sh, ss.QUERIES, 1, SortType("docid"), oix=oix)
    assert t[ss.EMPTY] == 0 and t[7] == ss.EXACT_K and t[8] == ss.EXACT_K - 1
    assert all(t[q] > 0 for q in range(len(t)) if q != ss.EMPTY)
    carr, _, qarr, _ = compile_queries(ss.QUERIES)
    m = np.nonzero(oracle.match_bitmap(oix, carr, qarr, ss.ONLY_MISSING))[0]
    for col in (ss.C_I32, ss.C_I64, ss.C_F32, ss.C_F64, ss.C_ONE):
        assert not sh.column_has[col][m].any()
    tie = slice(TIE_LO, TIE_LO + ss.TIE_DOCS)
    for col, v in ss.TIE_VALUE.items():
        assert (sh.columns[col][tie] == v).all() and (sh.column_has[col] is None or sh.column_has[col][tie].all())


@pytest.mark.parametrize("st", SORTS, ids=ss.sort_id)
def test_every_sort(shard, st):
    sh, oix = shard
    assert_same(ss.want_oracle(sh, ss.QUERIES, 512, st, oix=oix), ss.want_fields(sh, ss.QUERIES, 512, st, oix=oix), ss.sort_id(st))


@pytest.mark.parametrize("st", SORTS, ids=ss.sort_id)
def test_page_walks(shard, st):
    """oracle pages at k = 97, each after the previous page's last FieldDoc, concatenate to the reference's order"""
    sh, oix = shard
    full = ss.want_fields(sh, ss.QUERIES, 6000, st, oix=oix)
    nq = len(ss.QUERIES)
    goal = [min(int(full[3][q]), 6000 if full[3][q] <= 6000 else K_WALK * WALK_PAGES) for q in range(nq)]
    got = [[] for _ in range(nq)]
    after = [None] * nq
    active = [q for q in range(nq) if goal[q] > 0]
    while active:
        d, v, c, t = ss.want_oracle(sh, [ss.QUERIES[q] for q in active], K_WALK, st, [after[q] for q in active], oix)
        nxt = []
        for i, q in enumerate(active):
            assert t[i] == full[3][q]
            got[q] += list(zip(d[i, :c[i]].tolist(), v[i, :c[i]].tolist()))
            if c[i] == K_WALK and len(got[q]) < goal[q]:
                after[q] = FieldDoc(int(d[i, c[i] - 1]), int(v[i, c[i] - 1]))
                nxt.append(q)
        active = nxt
    for q in range(nq):
        n = len(got[q])
        assert n >= goal[q], (q, n, goal[q])
        n = min(n, 6000)
        assert [g[0] for g in got[q][:n]] == full[0][q, :n].tolist(), (ss.sort_id(st), q)
        assert [g[1] for g in got[q][:n]] == full[1][q, :n].tolist(), (ss.sort_id(st), q)


@pytest.mark.parametrize("st", SORTS, ids=ss.sort_id)
def test_synthetic_afters(shard, st):
    sh, oix = shard
    qs, after = ss.synthetic_afters(sh, st, [ss.QUERIES[q] for q in (0, 1, 4, ss.ONLY_MISSING, 9)],
                                    [DOC_BASE - 7, DOC_BASE + N // 2, DOC_BASE + 1234, DOC_BASE + N + 9])
    assert_same(ss.want_oracle(sh, qs, 40, st, after, oix), ss.want_fields(sh, qs, 40, st, after, oix), ss.sort_id(st))


# ---- hand-made 20-doc leaves ----

MISSING_DOCS = [2, 5, 7, 9, 12, 15]


def leaf(values, doc_base=100):
    n = len(values)
    sh = ix.HostShard(n, doc_base, np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros(0, np.int32), [ix.TextField(None, n, n)])
    has = np.ones(n, np.uint8)
    has[MISSING_DOCS] = 0
    sh.columns, sh.column_has = [np.asarray(values, np.int64)], [has]
    return sh


F = float_to_sortable_int
FLOATS = [F(x) for x in (3.0, -1.0, 0.0, 8.5, 2.0, 0.0, -7.0, 1.0, 4.0, 0.0, 9.0, 3.0, 0.0, 6.0, -2.0, 0.0, 5.0, 1.0, 3.0, -0.0)]
INTS = [4, -3, 0, 8, 2, 0, -7, 1, 4, 0, 9, 3, 0, 6, -2, 0, 5, 1, 3, -(2**31)]   # doc 19 holds INT32_MIN


def expected(values, st, after_doc):
    """local docs strictly after (missing value, after_doc), in sort order: Python tuples (signed value, doc)"""
    m = st.missing_value()
    sign = -1 if st.reverse else 1
    rows = sorted((sign * (m if d in MISSING_DOCS else v), d) for d, v in enumerate(values))
    return [d for key, d in rows if (key, d) > (sign * m, after_doc)]


@pytest.mark.parametrize("values,st,after_7", [
    # missing +inf, held by no doc: the missing group sorts first, and the page continues inside it
    (FLOATS, SortType(0, True, True, "float"), [9, 12, 15, 10, 3, 13, 16, 8, 0, 11, 18, 4, 17]),
    # missing -inf, held by no doc
    (FLOATS, SortType(0, False, False, "float"), [9, 12, 15, 6, 14, 1, 19, 17]),
    # missing INT32_MIN, held by doc 19: it ties with the missing docs
    (INTS, SortType(0, False, False, "int"), [9, 12, 15, 19, 6, 1, 14]),
], ids=["float-desc-last", "float-asc-first", "int-asc-first-held"])
def test_after_the_missing_value_continues_inside_the_missing_group(values, st, after_7):
    sh = leaf(values)
    docs = (7, -1, 19, 25)   # inside the group, below and above the leaf
    qs = [MatchAllDocsQuery()] * len(docs)
    after = [FieldDoc(sh.doc_base + d, st.missing_value()) for d in docs]
    assert expected(values, st, 7)[:len(after_7)] == after_7
    for d, v, c, t in (ss.want_oracle(sh, qs, 20, st, after), ss.want_fields(sh, qs, 20, st, after)):
        assert (t == 20).all()
        for i, a in enumerate(docs):
            assert (d[i, :c[i]] - sh.doc_base).tolist() == expected(values, st, a), (i, a)
            miss = np.isin(d[i, :c[i]] - sh.doc_base, MISSING_DOCS)
            assert (v[i, :c[i]][miss] == st.missing_value()).all()
