"""Reference for sorted top hits (TopHitsCollector with a querySort: TopHitsCollectorManager.java:126-162 over Lucene's
TopFieldCollector), the checker of nrtgpu_search_bool_aggs_sorted_hits. TEST INFRASTRUCTURE ONLY.

A collector's bucket is a set of matching live docs (a terms bucket, the docs that pass a filter, or every doc a query
collects) with the scores the top-level hit list gives them. Its hits are ordered by the Sort with
sort_fields_reference's comparator (field_values / field_keys / deciding: columns with missing values and MIN / MAX
selectors, the global doc id, a leading score), the last tie-break the global doc id ascending, as a numpy lexsort;
positions [start_hit, top_hits) are returned with their FieldDoc values. Without a Sort the order is score descending,
then global doc ascending. Fields are (kind, column, reverse, selector, missing_value) tuples."""
import numpy as np

import sort_fields_reference as sfr


def top_hits(sh, docs, scores, fields, top, start):
    """(global docs, FieldDoc values int64 [n, n_fields] or None without a Sort) of positions [start, top) of the bucket
    whose local doc ids are `docs`, with float32 `scores` per doc"""
    docs = np.asarray(docs, np.int64)
    scores = np.asarray(scores, np.float32)
    gdoc = docs + sh.doc_base
    if fields is None:
        order = np.lexsort((gdoc, -scores.astype(np.float64)))[:top][start:]
        return gdoc[order], None
    sfr.check_fields(sh, fields)
    ne = sfr.deciding(fields)
    fv = [sfr.field_values(sh, f, docs, scores) for f in fields]
    keys = [sfr.field_keys(f, v) for f, v in zip(fields[:ne], fv[:ne])]
    order = np.lexsort([gdoc] + [k for k in reversed(keys)])[:top][start:]
    return gdoc[order], np.stack([np.asarray(v, np.int64)[order] for v in fv], axis=1).reshape(len(order), len(fields))
