"""Reference for sorts of several fields (Lucene TopFieldCollector over a Sort of 1..8 SortFields; reference SortParser.java:54-92,
Sortable.java:34-45, NumberFieldDef.java:266-278), the checker of nrtgpu_search_sorted_fields. TEST INFRASTRUCTURE ONLY.

It is built on the oracle's own matching and scoring (oracle.match_bitmap: every matching live doc; oracle.score_docs: the
scores orc_search gives them), so a SCORE field holds exactly the oracle's scores; the ordering is a numpy lexsort:
  - field kinds: 1 a numeric doc-value column (sortable-long domain; selector 0 MIN / 1 MAX on a multi-valued column, a doc
    without a value sorts as missing_value), 2 the doc id, 3 the score (first position only; higher first unless reverse);
  - fields after the first doc id cannot decide anything; the last tie-break is the global doc id, ascending;
  - FieldDoc values: the column's selected value or missing_value, the global doc id, the score's float bits;
  - searchAfter (PagingFieldCollector): a hit qualifies iff (fields, doc) sorts strictly after (after values, after_doc).
Fields are (kind, column, reverse, selector, missing_value) tuples."""
import numpy as np

import oracle

COLUMN, DOCID, SCORE = 1, 2, 3
_SIGN = np.uint64(1 << 63)


def check_fields(sh, fields):
    if not 1 <= len(fields) <= 8:
        raise ValueError("a Sort has 1 to 8 fields")
    for i, (kind, col, _, sel, _) in enumerate(fields):
        if kind not in (COLUMN, DOCID, SCORE) or (kind == SCORE and i > 0):
            raise ValueError(f"sort field {i}: bad kind {kind}")
        if kind == COLUMN and (not 0 <= col < len(sh.columns) or sel not in (0, 1)):
            raise ValueError(f"sort field {i}: bad column {col} or selector {sel}")


def deciding(fields):
    """the fields that can decide the order: up to the first doc id, inclusive"""
    for i, f in enumerate(fields):
        if f[0] == DOCID:
            return i + 1
    return len(fields)


def field_values(sh, f, docs, scores):
    """int64 FieldDoc values of one field for local doc ids `docs` with their scores"""
    kind, col, _, sel, missing = f
    if kind == DOCID:
        return docs.astype(np.int64) + sh.doc_base
    if kind == SCORE:
        return np.asarray(scores, np.float32).view(np.uint32).astype(np.int64)
    vals = np.asarray(sh.columns[col], np.int64)
    offs = getattr(sh, "column_offsets", None) or []
    off = offs[col] if col < len(offs) else None
    if off is not None:
        a, b = off[docs], off[docs + 1]
        pick = np.clip(np.where(sel == 1, b - 1, a), 0, max(len(vals) - 1, 0))
        got = vals[pick] if len(vals) else np.zeros(len(docs), np.int64)
        return np.where(a == b, np.int64(missing), got)
    has = sh.column_has[col] if col < len(sh.column_has) else None
    v = vals[docs]
    return v if has is None else np.where(np.asarray(has)[docs] != 0, v, np.int64(missing))


def field_keys(f, values):
    """uint64 keys that ascend in sort order"""
    values = np.asarray(values, np.int64)
    if f[0] == SCORE:
        bits = values.astype(np.uint32)
        ordered = np.where(bits & np.uint32(0x80000000), ~bits, bits | np.uint32(0x80000000)).astype(np.uint64)
        return ordered if f[2] else ~ordered
    k = values.view(np.uint64) ^ _SIGN
    return ~k if f[2] else k


def search_sorted_fields(sh, carr, ncl, qarr, nq, top_k, fields, after_values=None, oix=None):
    """docs [nq, k] (global), values [nq, k, n_fields] int64, counts [nq], total hits [nq] (exact)"""
    check_fields(sh, fields)
    oix = oix or oracle.OracleIndex(sh)
    nf, ne = len(fields), deciding(fields)
    docs = np.zeros((nq, top_k), np.int32)
    vals = np.zeros((nq, top_k, nf), np.int64)
    counts = np.zeros(nq, np.int32)
    total = np.zeros(nq, np.int64)
    for q in range(nq):
        m = np.nonzero(oracle.match_bitmap(oix, carr, qarr, q))[0]
        total[q] = len(m)
        if not len(m):
            continue
        scores = np.zeros(len(m), np.float32)
        if any(f[0] == SCORE for f in fields):
            one = (type(qarr[q]) * 1)(qarr[q])
            _, s = oracle.score_docs(oix, carr, one, 1, (m + sh.doc_base)[None, :].astype(np.int32))
            scores = s[0]
        fv = [field_values(sh, f, m, scores) for f in fields]
        keys = [field_keys(f, v) for f, v in zip(fields[:ne], fv[:ne])]
        gdoc = m.astype(np.int64) + sh.doc_base
        keep = np.ones(len(m), bool)
        if after_values is not None and qarr[q].has_after:
            av = np.asarray(after_values[q], np.int64).reshape(-1)
            gt, eq = np.zeros(len(m), bool), np.ones(len(m), bool)
            for f, k, a in zip(fields[:ne], keys, av[:ne]):
                ak = field_keys(f, [a])[0]
                gt |= eq & (k > ak)
                eq &= k == ak
            keep = gt | (eq & (gdoc > qarr[q].after_doc))
        idx = np.nonzero(keep)[0]
        order = idx[np.lexsort([gdoc[idx]] + [k[idx] for k in reversed(keys)])][:top_k]
        n = len(order)
        counts[q] = n
        docs[q, :n] = gdoc[order]
        for j in range(nf):
            vals[q, :n, j] = fv[j][order]
    return docs, vals, counts, total
