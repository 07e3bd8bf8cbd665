"""Reference for the second pass of tree and phrase rescore queries (nrtgpu_score_docs_tree / nrtgpu_rescore_query_tree).
TEST INFRASTRUCTURE ONLY.

score_docs evaluates each query over the whole shard with tree_reference.evaluate and phrase_reference.PhraseLeaves, ANDs
the live docs, and reads the result at the query's own hits: an entry past counts[q], a doc outside the shard
[doc_base, doc_base + n_docs) or a deleted doc gets match 0 and score 0. rescore applies oracle.rescore_combine
(QueryRescore.combine + the re-sort) to that second pass and keeps min(count, window) hits."""
import numpy as np

import oracle
import phrase_reference as pr
import tree_reference as tr


def evaluate_all(sh, queries, oix=None, leaves=None):
    """(present bool [nq, n_docs], score float32 [nq, n_docs]) of every query over every doc, deletes applied"""
    from nrtsearch_b200.search import compile_tree
    carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq = compile_tree(queries, phrase_table=True)
    if leaves is None:
        leaves = pr.PhraseLeaves(sh, oix or oracle.OracleIndex(sh), parr, tarr)
    leaves.parr, leaves.tarr = parr, tarr   # (its phrase cache is keyed by the terms, not by the table)
    present = np.zeros((nq, sh.n_docs), bool)
    score = np.zeros((nq, sh.n_docs), np.float32)
    for q in range(nq):
        qq = qarr[q]
        p, s = tr.evaluate(sh, carr, narr, qq.clause_begin, qq.clause_end, qq.min_should_match, leaves)
        present[q] = p & leaves.live
        score[q] = np.where(present[q], s, np.float32(0))
    return present, score


def read_at_hits(sh, present, score, docs, counts=None):
    """matches uint8 [nq, n_hits], scores float32 [nq, n_hits] of the whole-shard evaluation at the hits docs (global ids)"""
    docs = np.asarray(docs, np.int64)
    nq, n = docs.shape
    local = docs - sh.doc_base
    ok = (local >= 0) & (local < sh.n_docs)
    if counts is not None:
        ok &= np.arange(n)[None, :] < np.asarray(counts)[:, None]
    li = np.where(ok, local, 0)
    rows = np.arange(nq)[:, None]
    m = ok & present[rows, li]
    return m.astype(np.uint8), np.where(m, score[rows, li], np.float32(0)).astype(np.float32)


def score_docs(sh, queries, docs, counts=None, oix=None, leaves=None):
    present, score = evaluate_all(sh, queries, oix, leaves)
    return read_at_hits(sh, present, score, docs, counts)


def rescore(docs, first, matches, second, counts, window, query_weight, rescore_weight):
    """docs, scores [nq, n_hits] and counts [nq] of the rescored lists (entries past a count are left as they were)"""
    d, s = np.array(docs, np.int32), np.array(first, np.float32)
    c = np.zeros(len(counts), np.int32)
    for q, n in enumerate(np.asarray(counts).tolist()):
        if n:
            d[q, :n], s[q, :n] = oracle.rescore_combine(docs[q, :n], first[q, :n], matches[q, :n], second[q, :n], query_weight,
                                                        rescore_weight)
        c[q] = min(n, window)
    return d, s, c
