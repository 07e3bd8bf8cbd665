"""References for NestedQuery (block joins), built on score_nodes_reference without changing it. TEST INFRASTRUCTURE ONLY.

  - NestedReference: score_nodes_reference.ScoreNodeReference (it walks the query objects) plus NestedQuery;
  - evaluate / search_tree / search: score_nodes_reference's array-level rules over compile_tree's arrays plus node kind
    NESTED (6), whose score mode is the node's min_should_match.

The rules (Lucene 10 ToParentBlockJoinQuery / BlockJoinScorer, as QueryNodeMapper.getNestedQuery builds it):
  - the parents are the docs of HostShard.parent_term; the child query BooleanQuery{FILTER path term, MUST query} is
    evaluated over every doc WITHOUT live docs (the child scorer does not read acceptDocs), the outer boosts folded into
    its leaves;
  - a matching child c joins the smallest parent > c; a child that is itself a parent, or follows the last parent, joins
    nothing;
  - a parent with n >= 1 joined children of float scores s_1..s_n (doc order) matches and scores NONE 0, SUM (float) of
    the double sum in doc order, AVG (float)(double sum / n), MAX / MIN the largest / smallest s_i; its own liveness
    applies on the page, as for every hit."""
import dataclasses

import numpy as np

import oracle
import phrase_reference as pr
import score_nodes_reference as snr
import tree_reference as tr
from nrtsearch_b200.search import NestedQuery, compile_tree
from query_reference import F32, fold_boost

NESTED = 6
NONE, AVG, MAX, MIN, SUM = 0, 1, 2, 3, 4
_MODES = {"none": NONE, "avg": AVG, "max": MAX, "min": MIN, "sum": SUM}


def parent_mask(sh) -> np.ndarray:
    """bool [n_docs]: the docs of the shard's parent term"""
    m = np.zeros(sh.n_docs, bool)
    if sh.parent_term is not None:
        t = int(sh.parent_term)
        m[sh.post_docs[int(sh.term_off[t]):int(sh.term_off[t + 1])]] = True
    return m


def join(present: np.ndarray, scores: np.ndarray, parents: np.ndarray, mode: int):
    """(present, score) of the parents over the children's (present, score), folded child after child in doc order"""
    n = len(parents)
    out_p, out_s = np.zeros(n, bool), np.zeros(n, np.float32)
    pdocs = np.nonzero(parents)[0]
    kids = np.nonzero(present & ~parents)[0]
    k = np.searchsorted(pdocs, kids, side="right")
    kids, k = kids[k < len(pdocs)], k[k < len(pdocs)]   # (children after the last parent join nothing)
    if len(kids) == 0:
        return out_p, out_s
    owner = pdocs[k]                       # non-decreasing: each parent's children are one run
    s = scores[kids].astype(np.float32)
    starts = np.concatenate([[0], np.nonzero(np.diff(owner))[0] + 1])
    cnt = np.diff(np.append(starts, len(kids)))
    par = owner[starts]
    out_p[par] = True
    if mode == NONE:
        return out_p, out_s
    if mode in (MAX, MIN):
        out_s[par] = (np.maximum if mode == MAX else np.minimum).reduceat(s, starts)
        return out_p, out_s
    dsum = np.add.reduceat(s.astype(np.float64), starts)   # runs of < 8 are summed in order by numpy
    for i in np.nonzero(cnt >= 8)[0]:                       # longer runs: in child order, one by one
        acc = 0.0
        for x in s[starts[i]:starts[i] + cnt[i]]:
            acc += float(x)
        dsum[i] = acc
    out_s[par] = (dsum if mode == SUM else dsum / cnt).astype(np.float32)
    return out_p, out_s


class NestedReference(snr.ScoreNodeReference):
    """ScoreNodeReference with NestedQuery at any depth (its node rules call eval)"""

    def __init__(self, sh):
        super().__init__(sh)
        self.parents = parent_mask(sh)

    def eval(self, q, boost=F32(1)):
        q, boost = fold_boost(q, boost)
        if isinstance(q, NestedQuery):
            if self.sh.parent_term is None:
                raise ValueError("index has no parent docs")
            p, s = self.eval(q.child_query(), boost)
            return join(p, s, self.parents, _MODES[q.score_mode])
        return super().eval(q, boost)


def evaluate(sh, carr, narr, begin, end, msm, leaves, parents, kind=tr.BOOL, node=None):
    """(present, score) over every doc of the node whose clauses are carr[begin:end] (node: its Node record, None for
    the root): score_nodes_reference.evaluate's rules plus NESTED"""
    children, occurs = [], []
    for i in range(begin, end):
        c = carr[i]
        if c.kind == tr.NODE:
            nd = narr[c.id]
            children.append(evaluate(sh, carr, narr, nd.clause_begin, nd.clause_end, nd.min_should_match, leaves, parents,
                                     nd.kind, nd))
        else:
            children.append(leaves(c))
        occurs.append(c.occur)
    if kind == NESTED:
        (p, s), = children
        return join(p, s, parents, node.min_should_match)
    if kind == tr.DISMAX:
        return tr._dismax_node(children, node.tie_breaker, sh.n_docs)
    if kind in (snr.CONSTANT, snr.MIN_SCORE):
        (p, s), = children
        if kind == snr.CONSTANT:
            return p, np.where(p, F32(node.boost), F32(0))
        ok = p & (s >= F32(node.min_score))
        return ok, np.where(ok, s * F32(node.boost), F32(0)).astype(np.float32)
    return tr._bool_node(children, occurs, msm, sh.n_docs)


def search_tree(sh, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, top_k, oix=None):
    """docs [nq, k] (global), scores [nq, k], counts [nq], total hits [nq] (exact), relation [nq] (0) of
    compile_tree(..., phrase_table=True)'s arrays"""
    # the leaves are evaluated over every doc (a join's children are, without live docs; every other match meets the
    # live docs on the page)
    live = np.ones(sh.n_docs, bool) if sh.live_docs is None else np.asarray(sh.live_docs) != 0
    if sh.live_docs is not None:
        sh = dataclasses.replace(sh, live_docs=None)
        oix = None
    oix = oix or oracle.OracleIndex(sh)
    leaves = pr.PhraseLeaves(sh, oix, parr, tarr)
    parents = parent_mask(sh)
    docs, scores = np.zeros((nq, top_k), np.int32), np.zeros((nq, top_k), np.float32)
    counts, total = np.zeros(nq, np.int32), np.zeros(nq, np.int64)
    for q in range(nq):
        qq = qarr[q]
        p, s = evaluate(sh, carr, narr, qq.clause_begin, qq.clause_end, qq.min_should_match, leaves, parents)
        m = np.nonzero(p & live)[0]
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


# ---------------------------------------------------------------- nested corpora

def build_nested_shard(n_parents, seed, vocab=400, lam=3.0, trailing=3, parents_on_path=2):
    """A shard of blocks (children first, then their parent) with positions: field 0 holds the text of every doc (term
    ids 0 .. vocab - 1, Zipf-like), field 1 the _nested_path terms: vocab is _root (every parent: parent_term), vocab + 1
    and vocab + 2 two child paths. Each parent has a Poisson(lam) number of children; `trailing` children follow the last
    parent (they join nothing), and `parents_on_path` parents also hold path vocab + 1 (a matching child that is a parent
    joins nothing). Returns (shard, paths)."""
    rng = np.random.default_rng(seed)
    root, paths = vocab, (vocab + 1, vocab + 2)
    zipf = 1.0 / np.arange(1, vocab + 1) ** 0.9
    zipf /= zipf.sum()
    kids = rng.poisson(lam, n_parents)
    n_docs = int(kids.sum()) + n_parents + trailing
    kind = np.zeros(n_docs, np.int8)   # 1: parent
    kind[np.cumsum(kids + 1) - 1] = 1
    lens = np.where(kind == 1, rng.integers(1, 12, n_docs), rng.integers(1, 9, n_docs))
    doc = np.repeat(np.arange(n_docs), lens)
    pos = np.arange(len(doc)) - np.repeat(np.cumsum(lens) - lens, lens)
    term = rng.choice(vocab, len(doc), p=zipf)
    pdocs = np.nonzero(kind == 1)[0]
    cdocs = np.nonzero(kind == 0)[0]
    ctrm = np.where(rng.random(len(cdocs)) < 0.7, paths[0], paths[1])
    ctrm[cdocs > pdocs[-1]] = paths[0]
    odd = rng.choice(pdocs, parents_on_path, replace=False) if parents_on_path else np.zeros(0, np.int64)
    doc = np.concatenate([doc, pdocs, cdocs, odd])
    term = np.concatenate([term, np.full(len(pdocs), root), ctrm, np.full(len(odd), paths[0])])
    pos = np.concatenate([pos, lens[pdocs] + 100, lens[cdocs] + 100, lens[odd] + 101])
    term_field = [0] * vocab + [1, 1, 1]
    sh = pr.shard_from_token_arrays(n_docs, term_field, 2, doc, term, pos)
    sh.columns = [rng.integers(0, 1_000_000, n_docs).astype(np.int64)]
    sh.column_has = [None]
    sh.parent_term = root
    return sh, paths


def block_cuts(sh, n_leaves, rng):
    """doc boundaries that split the shard into n_leaves leaves right after parents (blocks never straddle leaves)"""
    pdocs = np.nonzero(parent_mask(sh))[0]
    picks = np.sort(rng.choice(len(pdocs) - 1, n_leaves - 1, replace=False))
    return [0] + [int(pdocs[i]) + 1 for i in picks] + [sh.n_docs]
