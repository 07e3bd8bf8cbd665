"""References for ConstantScoreQuery and MinScoreQuery nodes, built on the existing ones without changing them. TEST
INFRASTRUCTURE ONLY.

  - ScoreNodeReference: query_reference.Reference (it walks the query objects) plus the two wrappers;
  - evaluate / search_tree / search: tree_reference's node rules over compile_tree's arrays (phrase leaves through
    phrase_reference.PhraseLeaves) plus node kinds CONSTANT (3) and MIN_SCORE (4).

The rules (QueryNodeMapper's ConstantScoreQuery and MinThresholdQuery with MinScoreWrapper):
  - ConstantScoreQuery: matches where its filter does and scores the boost folded down to it;
  - MinScoreQuery: its query is evaluated with boost 1 (its own BoostQuerys apply); a doc matches where that float score
    s >= min_score (a NaN threshold never holds) and scores s * the boost folded down to it, in float. A threshold of 0
    is its query under that boost (the mapper returns it unwrapped); a negative one is refused."""
import numpy as np

import oracle
import phrase_reference as pr
import tree_reference as tr
from nrtsearch_b200.search import ConstantScoreQuery, MinScoreQuery, compile_tree
from query_reference import F32, Reference, fold_boost

CONSTANT, MIN_SCORE = 3, 4


class ScoreNodeReference(Reference):
    """Reference with ConstantScoreQuery and MinScoreQuery (its BooleanQuery and DisjunctionMaxQuery rules call eval, so the
    wrappers are found at any depth)"""

    def eval(self, q, boost=F32(1)):
        q, boost = fold_boost(q, boost)
        if isinstance(q, ConstantScoreQuery):
            p, _ = self.eval(q.filter)
            return p, np.where(p, boost, F32(0)).astype(np.float32)
        if isinstance(q, MinScoreQuery):
            if q.min_score < 0:
                raise ValueError(f"bad min_score {q.min_score}")
            if q.min_score == 0:
                return self.eval(q.query, boost)
            p, s = self.eval(q.query)
            ok = p & (s >= F32(q.min_score))
            return ok, np.where(ok, s * boost, F32(0)).astype(np.float32)
        return super().eval(q, boost)


def evaluate(sh, carr, narr, begin, end, msm, leaves, kind=tr.BOOL, node=None):
    """(present, score) over every doc of the node whose clauses are carr[begin:end] (node: its Node record, None for
    the root)"""
    children, occurs = [], []
    for i in range(begin, end):
        c = carr[i]
        if c.kind == tr.NODE:
            nd = narr[c.id]
            children.append(evaluate(sh, carr, narr, nd.clause_begin, nd.clause_end, nd.min_should_match, leaves, nd.kind, nd))
        else:
            children.append(leaves(c))
        occurs.append(c.occur)
    if kind == tr.DISMAX:
        return tr._dismax_node(children, node.tie_breaker, sh.n_docs)
    if kind in (CONSTANT, MIN_SCORE):
        (p, s), = children
        if kind == CONSTANT:
            return p, np.where(p, F32(node.boost), F32(0))
        ok = p & (s >= F32(node.min_score))
        return ok, np.where(ok, s * F32(node.boost), F32(0)).astype(np.float32)
    return tr._bool_node(children, occurs, msm, sh.n_docs)


def search_tree(sh, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, top_k, oix=None):
    """docs [nq, k] (global), scores [nq, k], counts [nq], total hits [nq] (exact), relation [nq] (0) of
    compile_tree(..., phrase_table=True)'s arrays"""
    oix = oix or oracle.OracleIndex(sh)
    leaves = pr.PhraseLeaves(sh, oix, parr, tarr)
    docs, scores = np.zeros((nq, top_k), np.int32), np.zeros((nq, top_k), np.float32)
    counts, total = np.zeros(nq, np.int32), np.zeros(nq, np.int64)
    for q in range(nq):
        qq = qarr[q]
        p, s = evaluate(sh, carr, narr, qq.clause_begin, qq.clause_end, qq.min_should_match, leaves)
        m = np.nonzero(p & leaves.live)[0]
        total[q] = len(m)
        sc, gdoc = s[m], m.astype(np.int64) + sh.doc_base
        if qq.has_after:
            a = F32(qq.after_score)
            keep = (sc < a) | ((sc == a) & (gdoc > qq.after_doc))
            sc, gdoc = sc[keep], gdoc[keep]
        order = np.lexsort((gdoc, -sc.astype(np.float64)))[:top_k]
        counts[q] = len(order)
        docs[q, :len(order)], scores[q, :len(order)] = gdoc[order], sc[order]
    return docs, scores, counts, total, np.zeros(nq, np.uint8)


def search(sh, queries, top_k, search_after=None, oix=None):
    """search_tree over nrtsearch_b200.search query objects"""
    return search_tree(sh, *compile_tree(queries, search_after, phrase_table=True), top_k, oix)
