"""Reference for multi-phrase leaves of query trees (MultiPhraseQuery, MatchPhrasePrefixQuery; clause kind 6,
NRTGPU_MULTI_PHRASE), the checker of the device's union lists. TEST INFRASTRUCTURE ONLY.

Restated from Lucene 10's MultiPhraseQuery (createWeight, rewrite, UnionPostingsEnum) and the reference project's
src/main/java/com/yelp/nrtsearch/server/query/MatchPhrasePrefixQuery.java (createQueryFromTokenStream, rewrite,
getPrefixTerms); pinned in tests/test_multi_phrase_reference.py to the hit sets of the reference's
MatchPhrasePrefixQueryTest and MultiMatchPhrasePrefixQueryTest:
  - a position matches a doc when any of its alternatives occurs there; its positions in the doc are the merged positions
    of those alternatives, repeats kept, and phrase_reference's exact_freq / sloppy_freq run over them;
  - weight = boost * (float) of the double sum of the float idf of every term with df > 0, a term repeated at several
    positions counted each time (createWeight memoises TermStates per term but adds a TermStatistics per occurrence),
    position after position, ascending term id within a position (none: no match);
  - one position is the BooleanQuery of SHOULD TermQuerys over its alternatives: (float) of the double sum of each
    present alternative's float BM25 at boost * its idf. Lucene collects prefix expansions in a HashSet, so the order of
    that sum is unspecified; a double holds 53 significand bits and each term a 24-bit float, so the sum is exact (and
    every order gives the same bits) when the alternatives' scores in a doc span fewer than 2^(53 - 24 - 7) = 2^22 in
    magnitude for 128 terms. Scores of one prefix's expansions can span more (idf alone ranges over 2^28 on a 10M-doc
    shard), so the device sums in ascending term id order, the order a term dictionary seek enumerates the expansions,
    and this reference does the same;
  - expand_prefix is the adaptor's expansion: the sorted term dictionary seeked at the prefix, terms taken while they
    start with it, stopping at max_expansions (0: 50), per leaf and into one set over the leaves as getPrefixTerms does.
search / search_tree combine the leaves with score_nodes_reference's node rules (BOOL, DISMAX, CONSTANT, MIN_SCORE)."""
import ctypes as C

import numpy as np

import oracle
import phrase_reference as pr
import score_nodes_reference as snr
import tree_reference as tr
from nrtsearch_b200 import _native
from nrtsearch_b200.search import compile_tree

MULTI_PHRASE = 6
DEFAULT_MAX_EXPANSIONS = 50


def expand_prefix(dictionaries, prefix: bytes, max_expansions: int = 0):
    """getPrefixTerms over the leaves: dictionaries[l] is leaf l's sorted term list (bytes); returns the expanded terms
    (a set, as the reference's HashSet) in the order they were found"""
    limit = max_expansions if max_expansions > 0 else DEFAULT_MAX_EXPANSIONS
    found = []
    for terms in dictionaries:
        i = int(np.searchsorted(np.array(terms, dtype=object), prefix)) if terms else 0   # seekCeil
        while i < len(terms) and terms[i].startswith(prefix):
            if terms[i] not in found:
                found.append(terms[i])
            if len(found) >= limit:
                return found
            i += 1
    return found


class MultiPhraseLeaves(pr.PhraseLeaves):
    """phrase_reference.PhraseLeaves plus multi-phrase leaves (clause kind 6) of the phrase table parr / tarr"""

    def union_positions(self, terms, d):
        """the merged positions of the alternatives `terms` in doc d (repeats kept)"""
        out = []
        for t in terms:
            p, docs = self.term_postings(t)
            k = int(np.searchsorted(docs, d))
            if k < len(docs) and docs[k] == d:
                out.extend(self.positions(int(p[k])))
        return sorted(out)

    def __call__(self, c):
        if c.kind != MULTI_PHRASE:
            return super().__call__(c)
        ph = self.parr[c.id]
        groups = []   # (position, [terms])
        for i in range(ph.term_begin, ph.term_end):
            t, p = int(self.tarr[i].term), int(self.tarr[i].position)
            if groups and groups[-1][0] == p:
                groups[-1][1].append(t)
            else:
                groups.append((p, [t]))
        sh, n = self.sh, self.sh.n_docs
        present, score = np.zeros(n, bool), np.zeros(n, np.float32)
        if not groups:
            return present, score
        if len(groups) == 1:   # MultiPhraseQuery.rewrite: SHOULD TermQuerys
            alts = sorted(groups[0][1])
            if len(alts) == 1:
                return super().__call__(_native.Clause(c.occur, tr.TERM, alts[0], c.boost, 0, 0))
            total = np.zeros(n, np.float64)
            for t in alts:   # ascending term id
                p, s = super().__call__(_native.Clause(tr.SHOULD, tr.TERM, t, c.boost, 0, 0))
                present |= p
                total += np.where(p, s.astype(np.float64), 0.0)
            return present, np.where(present, total.astype(np.float32), np.float32(0))
        key = ("multi", tuple((p, tuple(ts)) for p, ts in groups), int(ph.slop), np.float32(c.boost).tobytes())
        if key in self.cache:
            return self.cache[key]
        f = int(sh.term_field[groups[0][1][0]]) if sh.term_field is not None else 0
        fld = sh.fields[f]
        df = sh.term_df if sh.term_df is not None else np.diff(sh.term_off)
        idf, any_df = 0.0, False
        for t in [t for _, ts in groups for t in sorted(ts)]:
            if int(df[t]) > 0:
                idf += float(oracle.bm25_idf(int(df[t]), fld.doc_count))
                any_df = True
        if any_df:
            weight = np.float32(np.float32(c.boost) * np.float32(idf))
            cand = None
            for _, ts in groups:
                docs = np.unique(np.concatenate([self.term_postings(t)[1] for t in ts]))
                cand = docs if cand is None else np.intersect1d(cand, docs, assume_unique=True)
            offsets = [p for p, _ in groups]
            cache = oracle.bm25_cache(fld.k1, fld.b, float(oracle.lib().orc_bm25_avgdl(fld.sum_total_term_freq, fld.doc_count)))
            cp = cache.ctypes.data_as(C.POINTER(C.c_float))
            for d in cand.tolist():
                fr = pr.phrase_freq([self.union_positions(ts, d) for _, ts in groups], offsets, int(ph.slop))
                if fr > 0:
                    present[d] = True
                    nb = int(fld.norms[d]) if fld.norms is not None else 1
                    score[d] = oracle.lib().orc_bm25_score(weight, float(fr), nb, cp)
        self.cache[key] = (present, score)
        return present, score


def search_tree(sh, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, top_k, oix=None, leaves=None):
    """docs [nq, k] (global), scores [nq, k], counts [nq], total hits [nq] (exact), relation [nq] (0) of
    compile_tree(..., phrase_table=True)'s arrays"""
    oix = oix or oracle.OracleIndex(sh)
    leaves = leaves or MultiPhraseLeaves(sh, oix, parr, tarr)
    docs, scores = np.zeros((nq, top_k), np.int32), np.zeros((nq, top_k), np.float32)
    counts, total = np.zeros(nq, np.int32), np.zeros(nq, np.int64)
    for q in range(nq):
        qq = qarr[q]
        p, s = snr.evaluate(sh, carr, narr, qq.clause_begin, qq.clause_end, qq.min_should_match, leaves)
        m = np.nonzero(p & leaves.live)[0]
        total[q] = len(m)
        sc, gdoc = s[m], m.astype(np.int64) + sh.doc_base
        if qq.has_after:
            a = np.float32(qq.after_score)
            keep = (sc < a) | ((sc == a) & (gdoc > qq.after_doc))
            sc, gdoc = sc[keep], gdoc[keep]
        order = np.lexsort((gdoc, -sc.astype(np.float64)))[:top_k]
        counts[q] = len(order)
        docs[q, :len(order)], scores[q, :len(order)] = gdoc[order], sc[order]
    return docs, scores, counts, total, np.zeros(nq, np.uint8)


def search(sh, queries, top_k, search_after=None, oix=None):
    """search_tree over nrtsearch_b200.search query objects (MultiPhraseQuery / MatchPhrasePrefixQuery leaves included)"""
    return search_tree(sh, *compile_tree(queries, search_after, phrase_table=True), top_k, oix)
