"""Reference for Sorts with keyword fields (Lucene TopFieldCollector over a Sort that holds SortField(STRING) or
SortedSetSortField, as AtomFieldDef.getSortField builds them), the checker of NRTGPU_SORT_KEYWORD. TEST INFRASTRUCTURE ONLY.

A plain restatement of the rules, independent of the library's codes and orders:
  - a keyword field picks one term per doc as bytes, or None when the doc has no value: a SORTED column its term; a
    SORTED_SET column, whose n ordinals are ascending, ords[0] (MIN), ords[n-1] (MAX), ords[(n-1)//2] (MIDDLE_MIN) or
    ords[n//2] (MIDDLE_MAX);
  - terms compare as bytes (Python's bytes order is BytesRef.compareTo); None sorts before every term when missing is 0
    (STRING_FIRST) and after every term when it is 1 (STRING_LAST); reverse reverses the whole comparison, None included;
  - numeric, doc id and leading score fields are sort_fields_reference's, on the oracle's matching and scoring;
  - ties go to the next field, then to the global doc id ascending; searchAfter (PagingFieldCollector): a hit qualifies
    iff its tuple sorts strictly after the after tuple, or ties with it and has a greater global doc; a keyword after
    value is bytes (held by any leaf or none) or None;
  - over several leaves (merge_pages) the leaves' pages merge by the same comparison (TopFieldDocs.merge).
Fields are (kind, column, reverse, selector, missing) tuples; KEYWORD = 5, column a keyword column of the shard
(HostShard.keyword_columns). FieldDoc values come back in an object array: bytes / None for keyword fields, int else."""
import functools

import numpy as np

import oracle
import sort_fields_reference as sfr

COLUMN, DOCID, SCORE, KEYWORD = 1, 2, 3, 5
MIN, MAX, MIDDLE_MIN, MIDDLE_MAX = 0, 1, 2, 3


def selected_ords(col, docs, selector: int) -> np.ndarray:
    """the ordinal of the term that sorts each of `docs` in keyword column col (index.KeywordColumn), -1: no value"""
    docs = np.asarray(docs, np.int64)
    if not col.multi_valued:
        return col.ords[docs].astype(np.int64)
    a, n = col.offsets[docs], col.offsets[docs + 1] - col.offsets[docs]
    j = {MIN: np.zeros_like(n), MAX: n - 1, MIDDLE_MIN: (n - 1) // 2, MIDDLE_MAX: n // 2}[selector]
    pick = np.clip(a + j, 0, max(len(col.ords) - 1, 0))
    got = col.ords[pick].astype(np.int64) if len(col.ords) else np.zeros(len(docs), np.int64)
    return np.where(n > 0, got, -1)


def selected_terms(col, docs, selector: int) -> np.ndarray:
    """the selected term of each of `docs` as bytes, or None (an object array)"""
    u, at = np.unique(selected_ords(col, docs, selector), return_inverse=True)
    terms = np.empty(len(u), object)
    terms[:] = [None if o < 0 else bytes(col.terms[int(o)]) for o in u]
    return terms[at.reshape(-1)]


def keyword_keys(f, terms, after=()):
    """int64 keys that ascend in the field's order for the terms (bytes / None) of some docs and after values: terms rank
    by bytes comparison, None below or above them all by the missing rule, then the whole under reverse"""
    _, _, reverse, _, missing = f
    held = sorted({t for t in set(terms) | set(after) if t is not None})
    at = {t: i for i, t in enumerate(held)}
    none = len(held) if missing else -1
    k = np.array([none if t is None else at[t] for t in terms], np.int64)
    ka = np.array([none if t is None else at[t] for t in after], np.int64)
    return (-k, -ka) if reverse else (k, ka)


def field_keys(f, values, after=()):
    """keys ascending in sort order of the FieldDoc values of one field (and of after values)"""
    if f[0] == KEYWORD:
        return keyword_keys(f, values, after)
    return sfr.field_keys(f, values), sfr.field_keys(f, list(after)) if len(after) else np.zeros(0, np.uint64)


def _fv(sh, f, docs, scores, kw_columns):
    if f[0] == KEYWORD:
        return selected_terms(kw_columns[f[1]], docs, f[3])
    return sfr.field_values(sh, f, docs, scores)


def _to_object(f, v):
    return v if f[0] == KEYWORD else np.asarray(v, np.int64).astype(object)


def search(sh, carr, ncl, qarr, nq, top_k, fields, after_values=None, oix=None, kw_columns=None, restrict=None):
    """docs [nq, k] (global), values [nq, k, n_fields] object, counts [nq], total hits [nq] (exact). restrict: a bool mask
    over the leaf's docs that the matches are cut to (the docs a filter collector passes, or a terms bucket holds)"""
    kw_columns = sh.keyword_columns if kw_columns is None else kw_columns
    oix = oix or oracle.OracleIndex(sh)
    nf, ne = len(fields), sfr.deciding(fields)
    docs = np.zeros((nq, top_k), np.int32)
    vals = np.full((nq, top_k, nf), None, object)
    counts = np.zeros(nq, np.int32)
    total = np.zeros(nq, np.int64)
    for q in range(nq):
        hit = oracle.match_bitmap(oix, carr, qarr, q)
        m = np.nonzero(hit if restrict is None else np.asarray(hit, bool) & restrict)[0]
        total[q] = len(m)
        if not len(m):
            continue
        scores = np.zeros(len(m), np.float32)
        if any(f[0] == SCORE for f in fields):
            one = (type(qarr[q]) * 1)(qarr[q])
            _, s = oracle.score_docs(oix, carr, one, 1, (m + sh.doc_base)[None, :].astype(np.int32))
            scores = s[0]
        fv = [_fv(sh, f, m, scores, kw_columns) for f in fields]
        after = after_values is not None and qarr[q].has_after
        av = list(after_values[q]) if after else None
        keys, akeys = [], []
        for j, f in enumerate(fields[:ne]):
            k, ka = field_keys(f, fv[j], [av[j]] if after else [])
            keys.append(k)
            akeys.append(ka)
        gdoc = m.astype(np.int64) + sh.doc_base
        keep = np.ones(len(m), bool)
        if after:
            gt, eq = np.zeros(len(m), bool), np.ones(len(m), bool)
            for k, ka in zip(keys, akeys):
                gt |= eq & (k > ka[0])
                eq &= k == ka[0]
            keep = gt | (eq & (gdoc > qarr[q].after_doc))
        idx = np.nonzero(keep)[0]
        order = idx[np.lexsort([gdoc[idx]] + [k[idx] for k in reversed(keys)])][:top_k]
        n = len(order)
        counts[q] = n
        docs[q, :n] = gdoc[order]
        for j, f in enumerate(fields):
            vals[q, :n, j] = _to_object(f, fv[j])[order]
    return docs, vals, counts, total


def compare(fields, a, b) -> int:
    """-1 / 0 / 1: FieldDoc tuple a against b under the Sort's deciding fields, one field at a time"""
    for f, x, y in zip(fields[:sfr.deciding(fields)], a, b):
        if f[0] == KEYWORD:
            if x is None or y is None:
                c = 0 if x is None and y is None else ((1 if f[4] else -1) if x is None else (-1 if f[4] else 1))
            else:
                c = (x > y) - (x < y)
            c = -c if f[2] else c
        else:
            kx, ky = (int(k) for k in sfr.field_keys(f, [x, y]))
            c = (kx > ky) - (kx < ky)
        if c:
            return c
    return 0


def _row_order(fields):
    return functools.cmp_to_key(lambda a, b: compare(fields, a[0], b[0]) or (a[1] > b[1]) - (a[1] < b[1]))


def merge_pages(pages, fields, top_k):
    """TopFieldDocs.merge of the leaves' pages (search() results of doc-range leaves) by compare(), ties by global doc:
    docs, values, counts, totals"""
    nq = len(pages[0][2])
    nf = len(fields)
    docs = np.zeros((nq, top_k), np.int32)
    vals = np.full((nq, top_k, nf), None, object)
    counts = np.zeros(nq, np.int32)
    total = sum(p[3] for p in pages)
    for q in range(nq):
        rows = sorted([(tuple(p[1][q, i]), int(p[0][q, i])) for p in pages for i in range(p[2][q])], key=_row_order(fields))
        rows = rows[:top_k]
        counts[q] = len(rows)
        for i, (v, d) in enumerate(rows):
            docs[q, i] = d
            vals[q, i, :] = v
    return docs, vals, counts, total
