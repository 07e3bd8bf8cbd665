"""The numpy TopFieldDocs.merge of tests/searcher_leaves.py, which the GPU searcher tests use as their restatement of
the merge, checked without a GPU: per-leaf pages of sort_fields_reference merged by it equal that reference on the whole
shard, for the leaf cuts and the Sorts of the GPU tests, with and without a searchAfter FieldDoc."""
import numpy as np
import pytest

import oracle
import searcher_leaves as sl
import sort_single_shard as ss
from nrtsearch_b200.search import FieldDoc

K = 40


@pytest.fixture(scope="module")
def shard(built):
    sh = ss.make_shard(sl.N, sl.DOC_BASE, sl.TIE_LO)
    cuts = sl.cuts()
    leaves = [sh.doc_range(a, b) for a, b in zip(cuts, cuts[1:])]
    return sh, oracle.OracleIndex(sh), [(l, oracle.OracleIndex(l)) for l in leaves]


@pytest.mark.parametrize("sid,fields", sl.all_sorts(), ids=[s for s, _ in sl.all_sorts()])
def test_merged_leaf_pages_equal_the_whole_shard(shard, sid, fields):
    sh, oix, leaves = shard
    rf = sl.ref_fields(fields)
    wd, wv, wc, wt = sl.reference(sh, ss.QUERIES, K, fields, oix=oix)
    # a searchAfter FieldDoc taken from the whole shard's page: the 10th hit of each query (or none)
    after = [FieldDoc(int(wd[q, 9]), 0, tuple(int(x) for x in wv[q, 9])) if wc[q] > 9 else None for q in range(len(wc))]
    wd2, wv2, wc2, wt2 = sl.reference(sh, ss.QUERIES, K, fields, after, oix)
    for aft, (d0, v0, c0, t0) in ((None, (wd, wv, wc, wt)), (after, (wd2, wv2, wc2, wt2))):
        pages = [sl.reference(l, ss.QUERIES, K, fields, aft, lo) for l, lo in leaves]
        assert np.array_equal(sum(p[3] for p in pages), t0), sid
        assert any(p[2][q] == 0 and c0[q] > 0 for p in pages for q in range(len(c0))), "no leaf without a match"
        for q in range(len(c0)):
            md, mv = sl.merge_sorted(rf, [(p[0][q], p[1][q], p[2][q]) for p in pages], K)
            assert len(md) == c0[q], (sid, q)
            assert md.tolist() == d0[q, :c0[q]].tolist(), (sid, q)
            assert mv.tolist() == v0[q, :c0[q]].tolist(), (sid, q)


def test_a_cut_lies_inside_the_tie_group():
    c = sl.cuts()
    assert any(sl.TIE_LO < x < sl.TIE_LO + ss.TIE_DOCS for x in c)
    assert min(np.diff(c)) == sl.TINY
