"""Reference for the nested collectors of a terms aggregation (reference CollectorCreator.java:73-126,
TermsCollectorManager.fillBucketResultByCount :430-480 and fillBucketResultByNestedOrder :930-994, TopHitsCollectorManager
.java:126-162), the checker of nrtgpu_search_bool_aggs_nested. TEST INFRASTRUCTURE ONLY.

Built on the oracle's matching and scoring, as tests/sort_fields_reference.py is (oracle.match_bitmap: every matching live
doc; oracle.score_docs: the scores orc_search gives them). A bucket holds the matching docs with a value in the parent
column, keyed by that stored value:
  - min / max / sum per bucket: aggs_reference over the bucket's docs with a value in the nested column (a bucket without
    one keeps the unset value; a sum is (expected, bound) as aggs_reference.sum_value gives it);
  - the buckets returned: by count (ties to the smaller key), or by a nested value under Double.compare (NaN above +inf,
    -0.0 below 0.0) in the order_desc direction, ties to the smaller key; other_counts are the docs of the others;
  - top hits per returned bucket: its docs by score descending, then global doc ascending, positions [start_hit, top_hits);
    total hits the bucket's count.
A nested collector is ("min" | "max" | "sum", column, value_type) or ("top_hits", top_hits, start_hit)."""
import math

import numpy as np

import aggs_reference as ar
import oracle


def compare_key(v):
    """a sort key of a double that orders as java.lang.Double.compare"""
    if math.isnan(v):
        return (2, 0.0, 0.0)
    return (1, v, math.copysign(1.0, v))


def metric(kind, values):
    """(value, sum bound) of a min / max / sum over the doubles of a bucket"""
    if kind == "max":
        return ar.max_value(values), 0.0
    if kind == "min":
        return ar.min_value(values), 0.0
    return ar.sum_value(values)


def order_buckets(keys, counts, size, order_desc=True, values=None):
    """indices of the returned buckets: by count, or by `values` (Double.compare) when given; ties to the smaller key"""
    idx = sorted(range(len(keys)), key=lambda b: keys[b])
    if values is None:
        idx.sort(key=lambda b: counts[b], reverse=order_desc)
    else:
        idx.sort(key=lambda b: compare_key(values[b]), reverse=order_desc)
    return idx[:size]


def top_hits(docs, scores, top, start):
    """global docs and scores of positions [start, top) by (score desc, doc asc)"""
    order = np.lexsort((docs, -np.asarray(scores, np.float64)))[:top]
    return docs[order][start:], np.asarray(scores, np.float32)[order][start:]


def terms_nested(sh, match, column, size, order_desc, nested, order_by=None, scores=None):
    """one query's terms result with nested collectors.
    match: bool [n_docs]; nested: {name: spec}; order_by: a name of nested or None; scores: float32 [n_docs] (top hits).
    Returns the terms dict of aggs_reference.terms_from_counts plus "nested": {name: [(value, bound)] per returned bucket
    | [(docs, scores, total_hits)] per returned bucket}."""
    col = np.asarray(sh.columns[column], np.int64)
    has = sh.column_has[column] if column < len(sh.column_has) else None
    sel = match if has is None else match & (np.asarray(has) != 0)
    docs = np.nonzero(sel)[0]
    keys, inv, cnt = np.unique(col[docs], return_inverse=True, return_counts=True)
    members = np.split(docs[np.argsort(inv, kind="stable")], np.cumsum(cnt)[:-1])   # each bucket's docs, ascending
    counts = cnt.tolist()

    def bucket_metric(spec, b):
        kind, c, vt = spec
        h = sh.column_has[c] if c < len(sh.column_has) else None
        d = members[b] if h is None else members[b][np.asarray(h)[members[b]] != 0]
        return metric(kind, ar.as_doubles(np.asarray(sh.columns[c], np.int64)[d], vt))

    values = None
    if order_by is not None:
        values = [bucket_metric(nested[order_by], b)[0] for b in range(len(keys))]
    chosen = order_buckets(keys.tolist(), counts, size, order_desc, values)
    n = len(chosen)
    out = {"keys": np.zeros(size, np.int64), "counts": np.zeros(size, np.int32), "n": n, "total_buckets": len(keys),
           "other_counts": int(sum(counts) - sum(counts[b] for b in chosen)), "nested": {}}
    out["keys"][:n] = keys[chosen]
    out["counts"][:n] = [counts[b] for b in chosen]
    for name, spec in nested.items():
        if spec[0] == "top_hits":
            res = []
            for b in chosen:
                g = members[b].astype(np.int64) + sh.doc_base
                d, s = top_hits(g, scores[members[b]], spec[1], spec[2])
                res.append((d, s, counts[b]))
            out["nested"][name] = res
        else:
            out["nested"][name] = [bucket_metric(spec, b) for b in chosen]
    return out


def query_scores(sh, oix, carr, qarr, q, match):
    """float32 [n_docs]: the oracle's score of every doc query q matches (0 elsewhere)"""
    s = np.zeros(sh.n_docs, np.float32)
    m = np.nonzero(match)[0]
    if len(m):
        one = (type(qarr[q]) * 1)(qarr[q])
        _, got = oracle.score_docs(oix, carr, one, 1, (m + sh.doc_base)[None, :].astype(np.int32))
        s[m] = got[0]
    return s
