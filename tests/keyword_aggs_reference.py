"""Reference for terms aggregations over keyword columns (reference OrdinalTermsCollectorManager.java: collect() counts
segmentOrdsMapping.get(ord) for a SORTED doc's ordinal and for every ordinal of a SORTED_SET doc, and hands the doc to the
nested collectors once per ordinal; TermsCollectorManager.fillBucketResultByCount :430-480 picks the buckets), the checker
of terms aggregations with value_type 3. TEST INFRASTRUCTURE ONLY.

A column is an index.KeywordColumn: a term dictionary in byte order and per-doc ordinals (a set per doc for SORTED_SET).
  - counts: each matching doc adds one to the bucket of each of its ordinals;
  - buckets: the `size` largest (order_desc) or smallest counts, ties to the smaller term in byte order, which is the
    smaller ordinal; totalBuckets the non-empty buckets, otherCounts the counts of the others (so over a SORTED_SET column
    the counts sum to the matching docs' values, not to the docs);
  - nested collectors: over a bucket's docs (a doc of several terms is in several buckets), as nested_aggs_reference;
  - several leaves: every leaf numbers its own dictionary; the reader-wide dictionary is the byte-order union, and a leaf's
    ordinal maps to its term's place in it (union, global_column)."""
import numpy as np

import aggs_reference as ar
import nested_aggs_reference as nr
from nrtsearch_b200.index import KeywordColumn


def union(columns):
    """the reader-wide dictionary of a keyword column over leaves: the byte-order union of their dictionaries"""
    return sorted({t for c in columns for t in c.terms})


def global_column(columns):
    """the column of the whole shard (leaves in order) numbered in the union of the leaves' dictionaries"""
    uni = union(columns)
    at = {t: i for i, t in enumerate(uni)}
    ords, offs, multi = [], [np.zeros(1, np.int64)], columns[0].multi_valued
    base = 0
    for c in columns:
        m = np.array([at[t] for t in c.terms] + [-1], np.int32)   # (index -1: no value)
        ords.append(m[c.ords])
        if multi:
            offs.append(c.offsets[1:] + base)
            base += int(c.offsets[-1])
    o = np.concatenate(ords) if ords else np.zeros(0, np.int32)
    return KeywordColumn(uni, o.astype(np.int32), np.concatenate(offs) if multi else None)


def doc_ords(col, docs):
    """(ordinal, doc) of every value of the given docs, in doc order"""
    if col.offsets is None:
        o = col.ords[docs]
        keep = o >= 0
        return o[keep].astype(np.int64), np.asarray(docs)[keep]
    lens = (col.offsets[1:] - col.offsets[:-1])[docs]
    first = col.offsets[docs]
    idx = np.repeat(first - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens) + np.arange(int(lens.sum()), dtype=np.int64)
    return col.ords[idx].astype(np.int64), np.repeat(np.asarray(docs), lens)


def counts(col, match):
    """int64 [n_terms]: the matching docs of each term's bucket"""
    o, _ = doc_ords(col, np.nonzero(match)[0])
    return np.bincount(o, minlength=len(col.terms)).astype(np.int64)


def terms(col, match, size, order_desc=True):
    """one query's result: {"keys" (str, the returned terms), "ords", "counts", "n", "total_buckets", "other_counts"}"""
    c = counts(col, match)
    present = np.nonzero(c)[0]
    chosen = [present[b] for b in nr.order_buckets(present.tolist(), c[present].tolist(), size, order_desc)]
    return {"keys": [col.terms[b].decode("utf-8") for b in chosen], "ords": np.array(chosen, np.int64),
            "counts": np.array([c[b] for b in chosen], np.int64), "n": len(chosen), "total_buckets": len(present),
            "other_counts": int(c.sum() - sum(c[b] for b in chosen))}


def terms_nested(sh, col, match, size, order_desc, nested, order_by=None, scores=None):
    """terms() with nested collectors (nested_aggs_reference's specs: ("min" | "max" | "sum", column, value_type) or
    ("top_hits", top_hits, start_hit)), a bucket's docs being those with its term; order_by: a nested min / max / sum
    that orders the buckets; scores: float32 [n_docs] (top hits). Adds "nested": {name: [(value, bound)] |
    [(docs, scores, total_hits)]} per returned bucket, and "members": the returned buckets' docs."""
    o, d = doc_ords(col, np.nonzero(match)[0])
    c = np.bincount(o, minlength=len(col.terms))
    present = np.nonzero(c)[0]
    members = {int(b): np.sort(d[o == b]) for b in present}

    def bucket_metric(spec, b):
        kind, cc, vt = spec
        h = sh.column_has[cc] if cc < len(sh.column_has) else None
        m = members[b] if h is None else members[b][np.asarray(h)[members[b]] != 0]
        return nr.metric(kind, ar.as_doubles(np.asarray(sh.columns[cc], np.int64)[m], vt))

    values = None if order_by is None else [bucket_metric(nested[order_by], int(b))[0] for b in present]
    chosen = [int(present[i]) for i in nr.order_buckets(present.tolist(), c[present].tolist(), size, order_desc, values)]
    out = {"keys": [col.terms[b].decode("utf-8") for b in chosen], "ords": np.array(chosen, np.int64),
           "counts": np.array([c[b] for b in chosen], np.int64), "n": len(chosen), "total_buckets": len(present),
           "other_counts": int(c.sum() - sum(c[b] for b in chosen)), "nested": {}, "members": [members[b] for b in chosen]}
    for name, spec in nested.items():
        if spec[0] == "top_hits":
            out["nested"][name] = [nr.top_hits(members[b].astype(np.int64) + sh.doc_base, scores[members[b]], spec[1], spec[2])
                                   + (int(c[b]),) for b in chosen]
        else:
            out["nested"][name] = [bucket_metric(spec, b) for b in chosen]
    return out
