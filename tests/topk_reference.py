"""Plain numpy restatement of the relevance top-k kernels: merge_slices_kernel and merge_pairs_kernel (bool_kernel.cuh),
flush_top_k (common.cuh), rrf_blend_kernel and rescore_combine_kernel (hybrid_kernel.cuh).

Pages are built from (score, doc) pairs, ordered score desc then doc asc (TopDocs.merge), never from the kernels' 64-bit
keys. The key encoding (make_keys) is restated separately and only builds the kernels' inputs and the thresholds, which
the engine defines as keys. Blends run in np.float32 scalar operations in retriever order, with the kernel's expressions;
the rescore combine runs in np.float64 and is then cast. A page of k slots holds its hits first; the slots past the count
hold doc 0 and score 0.0 (include/nrtgpu.h)."""
from __future__ import annotations

import numpy as np

INT32_MAX = 2**31 - 1
_U32 = np.uint64(0xFFFFFFFF)


def make_keys(scores, docs) -> np.ndarray:
    """(ordered float bits << 32) | ~doc: the kernels' key of each (score, doc) pair (batch_plan.h make_key)"""
    b = np.asarray(scores, np.float32).view(np.uint32).astype(np.uint64)
    o = np.where(b & np.uint64(0x80000000), ~b & _U32, b | np.uint64(0x80000000))
    return (o << np.uint64(32)) | (~np.asarray(docs, np.int32).view(np.uint32)).astype(np.uint64)


def order(scores, docs) -> np.ndarray:
    """indices of the pairs, best first: score desc, then doc asc"""
    return np.lexsort((np.asarray(docs, np.int64), -np.asarray(scores, np.float64)))


def page(scores, docs, k: int):
    """the best k pairs: (docs int32, scores float32), at most k of each"""
    o = order(scores, docs)[:k]
    return np.asarray(docs, np.int32)[o], np.asarray(scores, np.float32)[o]


def padded(docs, scores, k: int):
    """a page in k slots: its hits, then doc 0 and score 0.0"""
    d, s = np.zeros(k, np.int32), np.zeros(k, np.float32)
    d[:len(docs)], s[:len(scores)] = docs, scores
    return d, s


def at_or_above(scores, docs, t_score, t_doc) -> np.ndarray:
    """pairs that are not worse than the pair (t_score, t_doc)"""
    s, d = np.asarray(scores, np.float32), np.asarray(docs, np.int64)
    return (s > np.float32(t_score)) | ((s == np.float32(t_score)) & (d <= t_doc))


def merge_slices_page(scores, docs, counts, top_k: int, doc_base: int = 0, theta=None):
    """one query of merge_slices_kernel: lists scores / docs [n_lists, top_k] with counts [n_lists]; theta None or the
    pair (score, doc) of the published threshold key, below which pairs are dropped. Returns (global docs, scores)."""
    s, d = np.asarray(scores, np.float32), np.asarray(docs, np.int32)
    m = np.arange(s.shape[1])[None, :] < np.asarray(counts)[:, None]
    s, d = s[m], d[m]
    if theta is not None:
        keep = at_or_above(s, d, *theta)
        s, d = s[keep], d[keep]
    pd, ps = page(s, d, top_k)
    return (pd.astype(np.int64) + doc_base).astype(np.int32), ps


def merge_slices_flags(total_hits=None, pruned=None, terminated=None, terminate_after: int = 0, known_hits=None, nq: int = 1):
    """the per-query outputs of merge_slices_kernel besides the page: (terminated after the call or None, total, flags).
    A query whose counted hits exceed terminate_after (> 0) terminated early; the total is max(counted, known) only when
    the query was pruned; flags bit 0 = relation GTE (pruned or terminated), bit 1 = terminated early."""
    tot = np.zeros(nq, np.int64) if total_hits is None else np.asarray(total_hits, np.uint64).astype(np.int64)
    term_out = None
    term = np.zeros(nq, bool)
    if terminated is not None:
        term_out = np.asarray(terminated, np.int32).copy()
        if terminate_after > 0 and total_hits is not None:
            term_out[tot > terminate_after] = 1
        term = term_out != 0
    pr = np.zeros(nq, bool) if pruned is None else np.asarray(pruned) != 0
    total = tot.copy()
    if known_hits is not None and pruned is not None:
        kn = np.asarray(known_hits, np.uint64).astype(np.int64)
        total = np.where(pr & (kn > tot), kn, tot)
    flags = ((pr | term).astype(np.int32)) | (term.astype(np.int32) << 1)
    return term_out, total, flags


def merge_pairs(docs, scores, counts, top_k: int, totals=None, flags=None):
    """TopDocs.merge of n_lists pages per query: docs / scores [n_lists, nq, top_k], counts [n_lists, nq]. Returns
    (docs [nq, top_k], scores [nq, top_k], counts [nq], totals [nq] int64 summed or None, flags [nq] ORed or None)."""
    docs, scores, counts = np.asarray(docs, np.int32), np.asarray(scores, np.float32), np.asarray(counts)
    nl, nq, _ = docs.shape
    od, os_, oc = np.zeros((nq, top_k), np.int32), np.zeros((nq, top_k), np.float32), np.zeros(nq, np.int32)
    for q in range(nq):
        d = np.concatenate([docs[l, q, :counts[l, q]] for l in range(nl)])
        s = np.concatenate([scores[l, q, :counts[l, q]] for l in range(nl)])
        pd, ps = page(s, d, top_k)
        od[q], os_[q] = padded(pd, ps, top_k)
        oc[q] = len(pd)
    t = None if totals is None else np.asarray(totals, np.int64).sum(axis=0, dtype=np.int64)
    f = None if flags is None else np.bitwise_or.reduce(np.asarray(flags, np.int32), axis=0)
    return od, os_, oc, t, f


def flush(scores, docs, count: int, cap: int, top_k: int, dec: int, g_theta: int, theta: int):
    """flush_top_k: the best min(count, cap, top_k) of the first min(count, cap) pairs. Once top_k are kept, the k-th key
    minus dec is published: g_theta = max(g_theta, kth - dec). The CTA's theta is raised to g_theta either way.
    Returns (docs, scores, kept, g_theta, theta)."""
    n = min(count, cap)
    d, s = page(np.asarray(scores)[:n], np.asarray(docs)[:n], top_k)
    if len(d) == top_k:
        kth = int(make_keys(s[top_k - 1:top_k], d[top_k - 1:top_k])[0]) - dec
        g_theta = max(g_theta, kth)
    return d, s, len(d), g_theta, max(theta, g_theta)


def blend(mode: int, docs, counts, boosts, top_out: int, scores=None, rank_constant: int = 0):
    """one query of rrf_blend_kernel: docs (and scores) [R, top_in], counts [R]. mode 0: weighted RRF, a hit at rank i
    (0-based) of retriever r adds boost_r / (k + i + 1) (k = rank_constant, 60 when <= 0); modes 1 / 2 / 3: MAX / SUM /
    running AVG of score * boost. A doc's contributions combine in retriever order, in float32. Returns (docs, scores,
    total distinct docs)."""
    k = rank_constant if rank_constant > 0 else 60
    acc: dict = {}
    have: dict = {}
    for r in range(len(counts)):
        b = np.float32(boosts[r])
        for i in range(int(counts[r])):
            d = int(docs[r][i])
            w = b / np.float32(k + i + 1) if mode == 0 else np.float32(scores[r][i]) * b
            if d not in acc:
                acc[d], have[d] = w, 1
                continue
            s = acc[d]
            if mode in (0, 2):
                s = s + w
            elif mode == 1:
                s = s if s > w else w
            else:
                s = (s * np.float32(have[d]) + w) / np.float32(have[d] + 1)
            acc[d], have[d] = np.float32(s), have[d] + 1
    ds = np.fromiter(acc.keys(), np.int64, len(acc))
    ss = np.fromiter(acc.values(), np.float32, len(acc))
    pd, ps = page(ss, ds, top_out)
    return pd, ps, len(acc)


def rescore_combine(docs, scores, matches, second, query_weight: float, rescore_weight: float, count=None):
    """one query of rescore_combine_kernel: the first count hits (all when None) get (float)(qw * first + rw * second)
    in double, or (float)(qw * first) without a second-pass match, and are re-sorted; the slots past count keep the input."""
    docs, scores = np.asarray(docs, np.int32).copy(), np.asarray(scores, np.float32).copy()
    n = len(docs) if count is None else int(count)
    first = scores[:n].astype(np.float64)
    m = np.asarray(matches[:n]) != 0
    comb = np.where(m, np.float64(query_weight) * first + np.float64(rescore_weight) * np.asarray(second[:n], np.float64),
                    np.float64(query_weight) * first).astype(np.float32)
    pd, ps = page(comb, docs[:n], n)
    docs[:n], scores[:n] = pd, ps
    return docs, scores
