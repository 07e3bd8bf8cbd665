"""Leaves, Sorts and the numpy TopFieldDocs.merge for the searcher tests over several leaves
(tests/test_gpu_searcher_leaves.py, tests/test_searcher_leaves_reference.py).

The shard is sort_single_shard.make_shard (8 % deletes, a 3,000-doc tie group on every sortable column) cut into uneven
doc-range leaves: one cut inside the tie group, so ties are decided across leaves by the global doc; one leaf of a few
dozen docs, on which most queries match nothing; and leaves of a few hundred thousand docs."""
from __future__ import annotations

import numpy as np

import sort_fields_reference as ref
import sort_single_shard as ss
from nrtsearch_b200.search import ScoreDoc, SortType, compile_queries

N, DOC_BASE = 600_000, 2_000
TIE_LO = 200_000
TINY = 37


def cuts(n=N, tie_lo=TIE_LO):
    """leaf boundaries (local docs): a cut inside the tie group, then a leaf of TINY docs"""
    mid = tie_lo + ss.TIE_DOCS // 2
    return [0, mid, mid + TINY, (mid + n) // 2 + 11_111, n]


def multi_sorts():
    """Sorts of several fields on the sort_single_shard columns: score first, MIN / MAX on the multi-valued column, DOCID
    last and in the middle, 8 fields"""
    ft = ss.FIELD_TYPE
    return {
        "score": [SortType("score")],
        "score-reverse,i32": [SortType("score", True), SortType(ss.C_I32, field_type=ft[ss.C_I32])],
        "score,mv-max,i64": [SortType("score"), SortType(ss.C_MV, selector="max", field_type="int"),
                             SortType(ss.C_I64, field_type="long")],
        "mv-min,i32-desc": [SortType(ss.C_MV, field_type="int"), SortType(ss.C_I32, True, field_type="int")],
        "mv-max-desc": [SortType(ss.C_MV, True, selector="max", field_type="int")],
        "one,f32-desc-last,docid": [SortType(ss.C_ONE, field_type="int"), SortType(ss.C_F32, True, True, "float"),
                                    SortType("docid")],
        "f64,docid-desc,i64": [SortType(ss.C_F64, field_type="double"), SortType("docid", True), SortType(ss.C_I64, field_type="long")],
        "8 fields": [SortType(ss.C_ONE, field_type="int"), SortType(ss.C_NONE, True, field_type="long"),
                     SortType(ss.C_MV, selector="max", field_type="int"), SortType(ss.C_I32_FULL, True, field_type="int"),
                     SortType(ss.C_F64, True, True, "double"), SortType(ss.C_I32, False, True, "int"),
                     SortType(ss.C_F32, field_type="float"), SortType("docid", True)],
    }


def all_sorts():
    """(id, fields) of every one-field Sort of sort_single_shard.sorts() and every multi-field Sort above"""
    out = [(ss.sort_id(st), [st]) for st in ss.sorts()]
    return out + list(multi_sorts().items())


def ref_fields(fields):
    return [tuple(getattr(f.c_field(), n) for n in ("kind", "column", "reverse", "selector", "missing_value")) for f in fields]


def reference(sh, qs, k, fields, after=None, oix=None):
    """sort_fields_reference.search_sorted_fields for SortTypes and FieldDocs: docs, values [nq, k, nf], counts, totals"""
    sd = None if after is None else [None if a is None else ScoreDoc(a.doc, 0.0) for a in after]
    carr, ncl, qarr, nq = compile_queries(qs, sd)
    av = None
    if after is not None:
        av = [[0] * len(fields) if a is None else list(a.values if a.values is not None else (a.value,)) for a in after]
    return ref.search_sorted_fields(sh, carr, ncl, qarr, nq, k, ref_fields(fields), av, oix)


def merge_sorted(fields, pages, k):
    """TopFieldDocs.merge of pages [(docs [k], values [k, nf], count)] under ref fields (kind, col, reverse, sel, missing):
    the fields up to the first DOCID decide, then the global doc ascending. Returns (docs, values [n, nf])."""
    nf = len(fields)
    docs = np.concatenate([np.asarray(p[0][:p[2]], np.int64) for p in pages])
    vals = np.concatenate([np.asarray(p[1][:p[2]], np.int64).reshape(-1, nf) for p in pages])
    ne = ref.deciding(fields)
    keys = [ref.field_keys(f, vals[:, j]) for j, f in enumerate(fields[:ne])]
    order = np.lexsort([docs] + list(reversed(keys)))[:k]
    return docs[order], vals[order]
