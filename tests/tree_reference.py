"""Reference for query trees (nested BooleanQuery and DisjunctionMaxQuery), the checker of nrtgpu_search_tree. TEST
INFRASTRUCTURE ONLY.

It is built on the oracle's own matching and scoring of single leaves: a leaf with its folded boost, as the one MUST clause
of a query, gives every doc's presence and float score (oracle.score_docs over the docs of a term's list, oracle.match_bitmap
for a range, every live doc for match-all: the score of a range or match-all leaf is its boost). The nodes are then combined
over all docs at once with numpy float32 / float64 arithmetic, by Lucene 10's rules:
  - BOOL: an absent MUST / FILTER clause or a present MUST_NOT clause rejects the doc; at least need_should SHOULD clauses
    must match (msm, or 1 when the node has no MUST / FILTER clause); the MUST and SHOULD sums are doubles added in clause
    order; a node without MUST / FILTER scores (float) should_sum, else req = (float) must_sum, and with a matching SHOULD
    clause req + (float) should_sum is a float add (msm == 0, ReqOptSumScorer) or a double add (msm > 0);
  - DISMAX: any matching disjunct; DisjunctionMaxScorer streams the disjuncts in clause order (a new max, score >= max, moves
    the old max into the double sum of the others) and scores (float)((double)max + others * (double)tie_breaker).
The page is a lexsort by (score desc, doc asc) after searchAfter; totalHits is exact (every match, searchAfter or not).
Input: the arrays nrtsearch_b200.search.compile_tree returns."""
import numpy as np

import oracle
from nrtsearch_b200 import _native

SHOULD, MUST, FILTER, MUST_NOT = 0, 1, 2, 3
TERM, RANGE, MATCH_ALL, NODE = 0, 1, 2, 3
BOOL, DISMAX = 0, 1


class LeafScores:
    """presence (bool [n_docs]) and float scores of leaves, cached per (kind, id, boost, lo, hi)"""

    def __init__(self, sh, oix):
        self.sh, self.oix, self.cache = sh, oix, {}
        self.live = np.ones(sh.n_docs, bool) if sh.live_docs is None else np.asarray(sh.live_docs) != 0

    def __call__(self, c):
        key = (c.kind, c.id, np.float32(c.boost).tobytes(), c.lo, c.hi)
        if key in self.cache:
            return self.cache[key]
        n = self.sh.n_docs
        clause = (_native.Clause * 1)(_native.Clause(MUST, c.kind, c.id, c.boost, c.lo, c.hi))
        query = (_native.Query * 1)(_native.Query(0, 1, 0, 0, 0, 0.0))
        present, score = np.zeros(n, bool), np.zeros(n, np.float32)
        if c.kind == TERM:
            docs = self.sh.post_docs[self.sh.term_off[c.id]:self.sh.term_off[c.id + 1]]
            if len(docs):
                m, s = oracle.score_docs(self.oix, clause, query, 1, (docs.astype(np.int64) + self.sh.doc_base)[None, :].astype(np.int32))
                present[docs] = m[0] != 0
                score[docs] = s[0]
        elif c.kind == RANGE:
            present = oracle.match_bitmap(self.oix, clause, query, 0) != 0
            score[:] = np.float32(c.boost)
        elif c.kind == MATCH_ALL:
            present = self.live.copy()
            score[:] = np.float32(c.boost)
        else:
            raise ValueError(f"bad leaf kind {c.kind}")
        score = np.where(present, score, np.float32(0))
        self.cache[key] = (present, score)
        return present, score


def _bool_node(children, occurs, msm, n):
    ok = np.ones(n, bool)
    must_sum, should_sum = np.zeros(n, np.float64), np.zeros(n, np.float64)
    n_should = np.zeros(n, np.int32)
    n_req = sum(o in (MUST, FILTER) for o in occurs)
    for (p, s), o in zip(children, occurs):
        if o in (MUST, FILTER):
            ok &= p
        if o == MUST_NOT:
            ok &= ~p
        if o == MUST:
            must_sum = np.where(p, must_sum + s.astype(np.float64), must_sum)
        if o == SHOULD:
            should_sum = np.where(p, should_sum + s.astype(np.float64), should_sum)
            n_should += p
    need = msm if msm > 0 else (1 if n_req == 0 else 0)
    ok &= n_should >= need
    if n_req == 0:
        score = should_sum.astype(np.float32)
    else:
        req, opt = must_sum.astype(np.float32), should_sum.astype(np.float32)
        both = (req.astype(np.float64) + opt.astype(np.float64)).astype(np.float32) if msm > 0 else req + opt
        score = np.where(n_should == 0, req, both)
    return ok, np.where(ok, score, np.float32(0))


def _dismax_node(children, tie, n):
    mx, other = np.zeros(n, np.float32), np.zeros(n, np.float64)
    any_ = np.zeros(n, bool)
    for p, s in children:
        ge = p & (s >= mx)
        other = np.where(ge, other + mx.astype(np.float64), np.where(p, other + s.astype(np.float64), other))
        mx = np.where(ge, s, mx)
        any_ |= p
    score = (mx.astype(np.float64) + other * np.float64(np.float32(tie))).astype(np.float32)
    return any_, np.where(any_, score, np.float32(0))


def evaluate(sh, carr, narr, begin, end, msm, leaves, kind=BOOL, tie=0.0):
    """(present, score) over every doc of the node whose clauses are carr[begin:end]"""
    children, occurs = [], []
    for i in range(begin, end):
        c = carr[i]
        if c.kind == NODE:
            nd = narr[c.id]
            children.append(evaluate(sh, carr, narr, nd.clause_begin, nd.clause_end, nd.min_should_match, leaves, nd.kind,
                                     nd.tie_breaker))
        else:
            children.append(leaves(c))
        occurs.append(c.occur)
    if kind == DISMAX:
        return _dismax_node(children, tie, sh.n_docs)
    return _bool_node(children, occurs, msm, sh.n_docs)


def search_tree(sh, carr, ncl, narr, nn, qarr, nq, top_k, oix=None):
    """docs [nq, k] (global), scores [nq, k], counts [nq], total hits [nq] (exact), relation [nq] (0)"""
    oix = oix or oracle.OracleIndex(sh)
    leaves = LeafScores(sh, oix)
    docs = np.zeros((nq, top_k), np.int32)
    scores = np.zeros((nq, top_k), np.float32)
    counts = np.zeros(nq, np.int32)
    total = np.zeros(nq, np.int64)
    for q in range(nq):
        qq = qarr[q]
        p, s = evaluate(sh, carr, narr, qq.clause_begin, qq.clause_end, qq.min_should_match, leaves)
        p &= leaves.live
        m = np.nonzero(p)[0]
        total[q] = len(m)
        sc = s[m]
        gdoc = m.astype(np.int64) + sh.doc_base
        if qq.has_after:
            a = np.float32(qq.after_score)
            keep = (sc < a) | ((sc == a) & (gdoc > qq.after_doc))
            sc, gdoc = sc[keep], gdoc[keep]
        order = np.lexsort((gdoc, -sc.astype(np.float64)))[:top_k]
        counts[q] = len(order)
        docs[q, :len(order)] = gdoc[order]
        scores[q, :len(order)] = sc[order]
    return docs, scores, counts, total, np.zeros(nq, np.uint8)


def search(sh, queries, top_k, search_after=None, oix=None):
    """search_tree over nrtsearch_b200.search query objects"""
    from nrtsearch_b200.search import compile_tree
    carr, ncl, narr, nn, qarr, nq = compile_tree(queries, search_after)
    return search_tree(sh, carr, ncl, narr, nn, qarr, nq, top_k, oix)

