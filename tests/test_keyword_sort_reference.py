"""The keyword sort reference (tests/keyword_sort_reference.py), the checker of tests/test_gpu_keyword_sort.py, pinned on the
CPU: against the reference's known answers (SortFieldTest.java:751-780, the 100-doc index's ATOM doc_id field, and
:1500-1670, the 10-doc sort_with_missing index), and against an independent restatement (brute: per-doc term selection
and stable per-field sorts written here, sharing no code with the reference) on a seeded leaf of about 100K docs with
SORTED and SORTED_SET columns, numeric ties, deletes, a leading score and searchAfter tuples; and the reference's merge of
doc-range leaves against the whole leaf."""
import numpy as np

import keyword_sort_reference as ref
import oracle
from nrtsearch_b200 import index as ix
from nrtsearch_b200.index import KeywordColumn
from nrtsearch_b200.search import (BooleanQuery, MatchAllDocsQuery, Occur, RangeQuery, ScoreDoc, SortType, TermQuery,
                                   compile_queries)

COLUMN, DOCID, SCORE, KEYWORD = 1, 2, 3, 5
INT_MIN = -(2**31)


def empty_shard(n, doc_base=0):
    sh = ix.HostShard(n, doc_base, np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros(0, np.int32), [ix.TextField(None, n, n)])
    sh.columns, sh.column_has, sh.column_offsets = [], [], []
    return sh


def missing_index():
    """SortFieldTest.initTestIndexWithMissing: doc i has int_field i (i < 5) or string_field str(9 - i) (i >= 5)"""
    sh = empty_shard(10)
    sh.columns = [np.array([i if i < 5 else 0 for i in range(10)], np.int64)]
    sh.column_has = [np.array([i < 5 for i in range(10)], np.uint8)]
    sh.column_offsets = [None]
    sh.keyword_columns = [KeywordColumn.from_values([None if i < 5 else str(9 - i) for i in range(10)], False)]
    return sh


def run(sh, fields, k, after=None, after_doc=0):
    sa = None if after is None else [ScoreDoc(after_doc, 0.0)]
    carr, ncl, qarr, nq = compile_queries([MatchAllDocsQuery()], sa)
    d, v, c, t = ref.search(sh, carr, ncl, qarr, nq, k, fields, None if after is None else [after])
    return d[0, :c[0]].tolist(), [tuple(x) for x in v[0, :c[0]]]


def INT(reverse):
    return (COLUMN, 0, int(reverse), 0, SortType(0, reverse, field_type="int").missing_value())


def STR(reverse):
    return (KEYWORD, 0, int(reverse), 0, 0)


def b(*xs):
    return [None if x is None else x.encode() for x in xs]


def test_sort_with_missing():   # testSortWithMissing and its three reversed variants
    sh = missing_index()
    cases = {
        (False, False): ([9, 8, 7, 6, 5, 0, 1, 2, 3, 4], [INT_MIN] * 5 + [0, 1, 2, 3, 4], b("0", "1", "2", "3", "4") + [None] * 5),
        (True, False): ([4, 3, 2, 1, 0, 9, 8, 7, 6, 5], [4, 3, 2, 1, 0] + [INT_MIN] * 5, [None] * 5 + b("0", "1", "2", "3", "4")),
        (False, True): ([5, 6, 7, 8, 9, 0, 1, 2, 3, 4], [INT_MIN] * 5 + [0, 1, 2, 3, 4], b("4", "3", "2", "1", "0") + [None] * 5),
        (True, True): ([4, 3, 2, 1, 0, 5, 6, 7, 8, 9], [4, 3, 2, 1, 0] + [INT_MIN] * 5, [None] * 5 + b("4", "3", "2", "1", "0")),
    }
    for (ir, sr), (ids, ints, strs) in cases.items():
        docs, vals = run(sh, [INT(ir), STR(sr)], 10)
        assert docs == ids, (ir, sr)
        assert [v[0] for v in vals] == ints and [v[1] for v in vals] == strs, (ir, sr)


def test_search_after_with_missing_sort_value():   # testSearchAfterWithMissingSortValue: both pages, a null after value
    sh = missing_index()
    fields = [STR(False), INT(True)]
    docs, vals = run(sh, fields, 3)
    assert docs == [4, 3, 2] and vals == [(None, 4), (None, 3), (None, 2)]
    docs, vals = run(sh, fields, 3, after=[None, 2], after_doc=2)
    assert docs == [1, 0, 9] and vals == [(None, 1), (None, 0), (b"0", INT_MIN)]


def doc_id_segments():
    """the 100-doc index of SortFieldTest.initTestIndex, ten segments of ten, its ATOM doc_id field (str(i) for doc i)"""
    out = []
    for s in range(10):
        sh = empty_shard(10, 10 * s)
        sh.keyword_columns = [KeywordColumn.from_values([str(i) for i in range(10 * s, 10 * s + 10)], False)]
        out.append(sh)
    return out


def test_doc_id_string_sort():   # testSortAtomDocId, testSortAtomDocIdSearchAfter: per segment, then merged
    fields = [STR(False)]
    for after, want in ((None, ["0", "1", "10", "11", "12"]), ([b"1"], ["1", "10", "11", "12", "13"])):
        pages = []
        for sh in doc_id_segments():
            sa = None if after is None else [ScoreDoc(0, 0.0)]   # LastHitInfo ("1") and last doc 0: the tie on "1" goes on
            carr, ncl, qarr, nq = compile_queries([MatchAllDocsQuery()], sa)
            pages.append(ref.search(sh, carr, ncl, qarr, nq, 5, fields, None if after is None else [after]))
        d, v, c, t = ref.merge_pages(pages, fields, 5)
        assert [x.decode() for x in v[0, :c[0], 0]] == want
        assert d[0, :c[0]].tolist() == [int(x) for x in want]
        assert t[0] == 100


# ---- the reference against an independent restatement on a seeded leaf ----

N, VOCAB = 100_000, 3_000


def seeded_shard(doc_base=0):
    sh = ix.synth_text_shard(N, VOCAB, min_len=4, poisson_mean=8.0)
    sh.doc_base = doc_base
    rng = np.random.default_rng(0x5EED)
    terms = ["", "a", "a\x00", "ab", "b", "café", "cafe", "\U0001f355", "z", "ÿ"] + [f"t{i:03d}" for i in range(60)]
    one = [None if rng.random() < 0.15 else terms[int(rng.integers(0, len(terms)))] for _ in range(N)]
    per = rng.integers(0, 6, N)
    sets = [[terms[int(x)] for x in rng.integers(0, len(terms), p)] for p in per]
    sh.keyword_columns = [KeywordColumn.from_values(one, False), KeywordColumn.from_values(sets, True)]
    sh.columns = [rng.integers(0, 5, N).astype(np.int64)]
    sh.column_has = [(rng.random(N) < 0.9).astype(np.uint8)]
    sh.column_offsets = [None]
    sh.live_docs = (rng.random(N) < 0.93).astype(np.uint8)
    return sh


def queries():
    return [MatchAllDocsQuery(), RangeQuery(0, 1, 3),
            BooleanQuery().add(TermQuery(3), Occur.SHOULD).add(TermQuery(7), Occur.SHOULD).add(TermQuery(20), Occur.SHOULD)]


SORTS = [
    [(KEYWORD, 0, 0, 0, 0)],
    [(KEYWORD, 0, 1, 0, 1)],
    [(KEYWORD, 1, 0, 2, 0), (COLUMN, 0, 1, 0, INT_MIN)],
    [(COLUMN, 0, 0, 0, INT_MIN), (KEYWORD, 1, 1, 3, 1)],
    [(SCORE, 0, 0, 0, 0), (KEYWORD, 0, 0, 0, 1)],
    [(KEYWORD, 0, 1, 0, 0), (DOCID, 0, 1, 0, 0)],
    [(KEYWORD, 0, 0, 0, 0), (KEYWORD, 1, 0, 1, 0)],
]


def own_term(col, d, selector):
    """doc d's sort term, read and chosen here without keyword_sort_reference: the doc's terms as bytes, sorted as bytes,
    then SortedSetSelector's pick (MIN the first, MAX the last, MIDDLE_MIN / MIDDLE_MAX the lower / upper middle)"""
    if not col.multi_valued:
        o = int(col.ords[d])
        return None if o < 0 else bytes(col.terms[o])
    ts = sorted(bytes(col.terms[int(o)]) for o in col.ords[int(col.offsets[d]):int(col.offsets[d + 1])])
    if not ts:
        return None
    return {0: ts[0], 1: ts[-1], 2: ts[(len(ts) - 1) // 2], 3: ts[len(ts) // 2]}[selector]


def own_value(sh, f, d, score):
    kind, col, _, sel, missing = f
    if kind == KEYWORD:
        return own_term(sh.keyword_columns[col], d, sel)
    if kind == DOCID:
        return d + sh.doc_base
    if kind == SCORE:
        return int(np.float32(score).view(np.uint32))
    has = sh.column_has[col]
    return int(sh.columns[col][d]) if has is None or has[d] else int(missing)


def brute(sh, oix, carr, qarr, q, fields, k, after=None):
    """the top k of query q restated without keyword_sort_reference: per-doc values from own_value, then stable Python
    sorts from the last deciding field to the first over (doc asc) order, each field with its own direction: a keyword by
    (missing group, bytes), where the group puts None before or after every term and reverse moves it too; a column by
    its sortable long; a score by its float, higher first; a doc id by its value. searchAfter: the after tuple joins the
    rows as a marker that sorts after a real row equal to it, and the rows after the marker qualify."""
    m = np.nonzero(oracle.match_bitmap(oix, carr, qarr, q))[0]
    scores = np.zeros(len(m), np.float32)
    if fields[0][0] == SCORE and len(m):
        one = (type(qarr[q]) * 1)(qarr[q])
        scores = oracle.score_docs(oix, carr, one, 1, (m + sh.doc_base)[None, :].astype(np.int32))[1][0]
    rows = [(tuple(own_value(sh, f, int(d), sc) for f in fields), int(d) + sh.doc_base, 0) for d, sc in zip(m, scores)]
    if after is not None:
        rows.append((tuple(after), qarr[q].after_doc, 1))
    rows.sort(key=lambda r: (r[1], r[2]))
    ne = next((i + 1 for i, f in enumerate(fields) if f[0] == DOCID), len(fields))
    for j in reversed(range(ne)):
        kind, _, reverse, _, missing = fields[j]
        if kind == KEYWORD:
            rows.sort(key=lambda r: (2 if missing else 0, b"") if r[0][j] is None else (1, r[0][j]), reverse=bool(reverse))
        elif kind == SCORE:
            rows.sort(key=lambda r: float(np.uint32(r[0][j]).view(np.float32)), reverse=not reverse)
        else:
            rows.sort(key=lambda r: r[0][j], reverse=bool(reverse))
    if after is not None:
        rows = rows[[r[2] for r in rows].index(1) + 1:]
    rows = rows[:k]
    return [r[1] for r in rows], [r[0] for r in rows]


def test_reference_equals_independent_restatement():
    sh = seeded_shard(doc_base=7)
    oix = oracle.OracleIndex(sh)
    qs = queries()
    for i, fields in enumerate(SORTS):   # (brute is slow: the match-all query under the first two Sorts only)
        carr, ncl, qarr, nq = compile_queries(qs)
        d, v, c, _ = ref.search(sh, carr, ncl, qarr, nq, 60, fields, oix=oix)
        for q in (range(nq) if i < 2 else range(1, nq)):
            wd, wv = brute(sh, oix, carr, qarr, q, fields, 60)
            assert d[q, :c[q]].tolist() == wd and [tuple(x) for x in v[q, :c[q]]] == wv, (fields, q)
        # searchAfter from the 30th hit, and from synthetic values: a term no doc holds, None and ""
        for q in (2,):
            if c[q] < 31:
                continue
            for after in (list(v[q, 30]), [b"a\x00\x00" if f[0] == KEYWORD else x for f, x in zip(fields, v[q, 30])],
                          [None if f[0] == KEYWORD else x for f, x in zip(fields, v[q, 30])],
                          [b"" if f[0] == KEYWORD else x for f, x in zip(fields, v[q, 30])]):
                sa = [ScoreDoc(int(d[q, 30]), 0.0)] * nq
                carr2, ncl2, qarr2, nq2 = compile_queries(qs, sa)
                d2, v2, c2, _ = ref.search(sh, carr2, ncl2, qarr2, nq2, 40, fields, [after] * nq2, oix=oix)
                wd, wv = brute(sh, oix, carr2, qarr2, q, fields, 40, after)
                assert d2[q, :c2[q]].tolist() == wd and [tuple(x) for x in v2[q, :c2[q]]] == wv, (fields, q, after)


def test_merge_of_doc_range_leaves_equals_whole():
    sh = seeded_shard()
    cuts = [0, 31_000, 77_000, N]
    leaves = [sh.doc_range(a, z) for a, z in zip(cuts, cuts[1:])]
    carr, ncl, qarr, nq = compile_queries(queries()[:2])
    for fields in SORTS[:4] + SORTS[5:]:
        whole = ref.search(sh, carr, ncl, qarr, nq, 50, fields)
        merged = ref.merge_pages([ref.search(l, carr, ncl, qarr, nq, 50, fields) for l in leaves], fields, 50)
        assert np.array_equal(whole[0], merged[0]) and np.array_equal(whole[2], merged[2]) and np.array_equal(whole[3], merged[3])
        assert all(tuple(a) == tuple(bb) for a, bb in zip(whole[1].reshape(-1, len(fields)), merged[1].reshape(-1, len(fields))))
