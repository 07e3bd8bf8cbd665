"""Reference for filter collectors (reference FilterCollectorManager.java), the checker of nrtgpu_search_bool_aggs_filtered.
TEST INFRASTRUCTURE ONLY.

Built on the oracle's matching, as tests/nested_aggs_reference.py is (oracle.match_bitmap: every matching live doc). The docs
of a filter are the query's matching docs that pass it (FilterCollectorManager.collect :353-360):
  - a query filter (QueryFilter :84-135): the docs the filter query matches, boosts and scores ignored (oracle.match_bitmap
    of the filter query; an empty BooleanQuery or one of MUST_NOT clauses only matches nothing);
  - a value set (SetQueryFilter :142-216): the docs with a value of the column, single- or multi-valued, whose stored
    sortable long is in the set (so floats and doubles compare by their bits: -0.0 != 0.0, NaN == NaN);
  - a filter under a filter: the docs that pass both.
docCount is their number; terms, min / max / sum and top hits under a filter are computed over exactly those docs, as
nested_aggs_reference computes them over a bucket's docs. A nested spec is ("terms", column, size, order_desc, nested,
order_by) | ("min" | "max" | "sum", column, value_type) | ("top_hits", top_hits, start_hit) | ("filter", mask, nested)."""
import numpy as np

import aggs_reference as ar
import nested_aggs_reference as nr
import oracle


def value_set_mask(sh, column, values) -> np.ndarray:
    """bool [n_docs]: the docs with a value of `column` in `values` (sortable longs)"""
    col = np.asarray(sh.columns[column], np.int64)
    s = np.asarray(list(values), np.int64)
    off = sh.column_offsets[column] if column < len(sh.column_offsets) else None
    if off is not None:
        c = np.concatenate([[0], np.cumsum(np.isin(col, s))])
        return c[np.asarray(off[1:])] > c[np.asarray(off[:-1])]
    has = sh.column_has[column] if column < len(sh.column_has) else None
    m = np.isin(col, s)
    return m if has is None else m & (np.asarray(has) != 0)


def query_mask(oix, carr, qarr, i) -> np.ndarray:
    """bool [n_docs]: the live docs filter query i matches"""
    return oracle.match_bitmap(oix, carr, qarr, i).astype(bool)


def filter_result(sh, sel, nested, scores=None) -> dict:
    """the result of a filter collector over the docs `sel` (bool [n_docs]: the query's matching docs that pass it):
    {"doc_count": int, name: a terms dict of nested_aggs_reference.terms_nested | (value, sum bound) | (docs, scores,
    total_hits) | a filter dict}. scores: float32 [n_docs] (top hits)."""
    out = {"doc_count": int(sel.sum())}
    for name, spec in nested.items():
        kind = spec[0]
        if kind == "terms":
            _, column, size, desc, sub, order_by = spec
            out[name] = nr.terms_nested(sh, sel, column, size, desc, sub, order_by, scores)
        elif kind == "filter":
            out[name] = filter_result(sh, sel & spec[1], spec[2], scores)
        elif kind == "top_hits":
            d = np.nonzero(sel)[0]
            gd, gs = nr.top_hits(d.astype(np.int64) + sh.doc_base, scores[d], spec[1], spec[2])
            out[name] = (gd, gs, len(d))
        else:
            _, column, vt = spec
            has = sh.column_has[column] if column < len(sh.column_has) else None
            d = np.nonzero(sel if has is None else sel & (np.asarray(has) != 0))[0]
            out[name] = nr.metric(kind, ar.as_doubles(np.asarray(sh.columns[column], np.int64)[d], vt))
    return out
