"""Object-level reference for every query engine: walks the query objects themselves (BooleanQuery, DisjunctionMaxQuery,
BoostQuery, TermQuery, RangeQuery, KeywordRangeQuery / KeywordPrefixQuery, MatchAllDocsQuery, PhraseQuery) over a
HostShard. TEST INFRASTRUCTURE ONLY.

It shares no code with the query compilers (search.compile_queries / compile_tree, batch_plan.inc) or with the oracle's
search, so a compiler mistake -- a boost folded in the wrong order, a node numbered wrongly, msm or a tie breaker put on
the wrong node, a clause dropped -- shows as a disagreement instead of being inherited by the judge.

  - BM25 (Lucene 10's BM25Similarity, k1 / b per field), in numpy float32 steps: idf = (float) log(1 + (N - df + 0.5) /
    (df + 0.5)) in double, df the index-wide docFreq (1 for an absent term); avgdl = (float) sumTotalTermFreq / docCount;
    cache[n] = 1 / (k1 * ((1 - b) + b * len(n) / avgdl)) over the 256 SmallFloat norm bytes (a field without norms reads
    byte 1); weight = boost * idf; score = weight - weight / (1 + freq * cache[norm]).
  - BoostQuery: boosts multiply outermost first in float, down to the leaves; a boost < 0, NaN or infinite is refused.
  - Constant-score leaves (ranges, keyword ranges and prefixes, match-all) score their boost. A numeric range matches a
    doc one of whose values lies in [lower, upper] (a doc without a value never matches); a keyword leaf compares terms
    as bytes (keyword_query_reference).
  - PhraseQuery: no terms matches nothing; one term is its TermQuery; else freq from phrase_reference's matchers (exact,
    or sloppy without repeats), weight = boost * (float) of the double sum of the terms' idf.
  - BooleanQuery: an absent MUST / FILTER clause or a present MUST_NOT clause rejects a doc; at least msm SHOULD clauses
    must match (1 when there is no MUST / FILTER clause). MUST and SHOULD scores are summed in double in clause order.
    Without MUST / FILTER the score is (float) should_sum; else req = (float) must_sum, and with a SHOULD clause matching,
    req + (float) should_sum is a float add at msm 0 (ReqOptSumScorer) and a double add at msm > 0 (ConjunctionScorer).
  - DisjunctionMaxQuery: any disjunct matches; the disjuncts stream in clause order (a score >= the max so far moves the
    old max into the double sum of the others) and score (float)((double) max + others * (double) tie_breaker).
  - The page: live matches after searchAfter (score < after, or equal and doc > after), ordered (score desc, doc asc);
    totalHits counts every live match."""
import math

import numpy as np

import keyword_query_reference as kqr
import phrase_reference as pr
from nrtsearch_b200.search import (BooleanQuery, BoostQuery, DisjunctionMaxQuery, KeywordPrefixQuery, KeywordRangeQuery,
                                   MatchAllDocsQuery, Occur, PhraseQuery, RangeQuery, TermQuery)

F32 = np.float32


def byte4_to_int(b: int) -> int:
    """SmallFloat.byte4ToInt"""
    if b < 24:
        return b
    i = b - 24
    bits, shift = i & 7, (i >> 3) - 1
    return 24 + (bits if shift == -1 else (bits | 8) << shift)


def idf(df: int, doc_count: int) -> np.float32:
    df = max(int(df), 1)
    return F32(math.log(1.0 + (float(doc_count) - float(df) + 0.5) / (float(df) + 0.5)))


def length_cache(k1: float, b: float, avgdl: np.float32) -> np.ndarray:
    lens = np.array([byte4_to_int(i) for i in range(256)], np.float32)
    k1, b = F32(k1), F32(b)
    t = (b * lens) / avgdl
    t = (F32(1) - b) + t
    return (F32(1) / (k1 * t)).astype(np.float32)


def bm25(weight: np.float32, freq: np.ndarray, norm: np.ndarray, cache: np.ndarray) -> np.ndarray:
    x = F32(1) + freq.astype(np.float32) * cache[norm]
    return (weight - weight / x).astype(np.float32)


def fold_boost(q, boost: np.float32):
    """(the query under its BoostQuerys, the boost folded outermost first in float)"""
    while isinstance(q, BoostQuery):
        if q.boost < 0 or not math.isfinite(q.boost):
            raise ValueError(f"bad boost {q.boost}")
        boost = F32(boost * F32(q.boost))
        q = q.query
    return q, boost


class Reference:
    """presence (bool [n_docs]) and float32 score [n_docs] of query objects over one HostShard"""

    def __init__(self, sh):
        self.sh, self.n = sh, sh.n_docs
        self.live = np.ones(sh.n_docs, bool) if sh.live_docs is None else np.asarray(sh.live_docs) != 0
        self.df = sh.term_df if sh.term_df is not None else np.diff(sh.term_off)
        self.caches = []
        for f in sh.fields:
            avgdl = F32(float(f.sum_total_term_freq) / float(f.doc_count))
            self.caches.append(length_cache(f.k1, f.b, avgdl))
        self.pstart = None
        self.memo = {}
        self.max_memo = max(16, (1 << 30) // (5 * sh.n_docs + 1))   # leaf arrays kept: about 1 GB

    def field_of(self, t: int) -> int:
        return 0 if self.sh.term_field is None else int(self.sh.term_field[t])

    def norms(self, f: int, docs: np.ndarray) -> np.ndarray:
        nb = self.sh.fields[f].norms
        return np.ones(len(docs), np.int64) if nb is None else nb[docs].astype(np.int64)

    # ------------------------------------------------------------ leaves

    def term(self, t: int, boost: np.float32):
        sh = self.sh
        a, b = int(sh.term_off[t]), int(sh.term_off[t + 1])
        docs, freqs = sh.post_docs[a:b], sh.post_freqs[a:b]
        f = self.field_of(t)
        w = F32(boost * idf(self.df[t], sh.fields[f].doc_count))
        present, score = np.zeros(self.n, bool), np.zeros(self.n, np.float32)
        present[docs] = True
        score[docs] = bm25(w, freqs, self.norms(f, docs), self.caches[f])
        return present, score

    def range_(self, q: RangeQuery):
        sh = self.sh
        col = np.asarray(sh.columns[q.column])
        off = sh.column_offsets[q.column] if q.column < len(sh.column_offsets) else None
        if off is None:
            present = (col >= q.lower) & (col <= q.upper)
            has = sh.column_has[q.column] if q.column < len(sh.column_has) else None
            if has is not None:
                present &= np.asarray(has) != 0
            return present
        inside = (col >= q.lower) & (col <= q.upper)
        owner = np.repeat(np.arange(self.n), np.diff(np.asarray(off)))
        return np.bincount(owner[inside], minlength=self.n) > 0

    def keyword(self, q):
        col = self.sh.keyword_columns[q.column]
        if isinstance(q, KeywordPrefixQuery):
            pred = kqr.prefix_pred(_bytes(q.prefix))
        else:
            pred = kqr.range_pred(None if q.lower is None else _bytes(q.lower), None if q.upper is None else _bytes(q.upper),
                                  q.include_lower, q.include_upper)
        hit = np.array([pred(bytes(t)) for t in col.terms] + [False], bool)   # ordinal -1 (no value) reads False
        if not col.multi_valued:
            return hit[np.asarray(col.ords)]
        owner = np.repeat(np.arange(self.n), np.diff(np.asarray(col.offsets)))
        return np.bincount(owner[hit[np.asarray(col.ords)]], minlength=self.n) > 0

    def phrase(self, q: PhraseQuery, boost: np.float32):
        sh = self.sh
        terms = sorted(q.term_positions(), key=lambda t: t[1])   # stable: the lead is the first of the smallest position
        if not terms:
            return np.zeros(self.n, bool), np.zeros(self.n, np.float32)
        if len(terms) == 1:
            return self.term(terms[0][0], boost)
        f = self.field_of(terms[0][0])
        s = 0.0
        for t, _ in terms:
            s += float(idf(self.df[t], sh.fields[f].doc_count))
        w = F32(boost * F32(s))
        if self.pstart is None:
            self.pstart = np.zeros(len(sh.post_freqs) + 1, np.int64)
            np.cumsum(sh.post_freqs, out=self.pstart[1:])
        lists = [(np.arange(sh.term_off[t], sh.term_off[t + 1]), sh.post_docs[sh.term_off[t]:sh.term_off[t + 1]]) for t, _ in terms]
        cand = lists[0][1]
        for _, d in lists[1:]:
            cand = np.intersect1d(cand, d, assume_unique=True)
        offsets = [p for _, p in terms]
        present, score = np.zeros(self.n, bool), np.zeros(self.n, np.float32)
        if len(cand):
            if q.slop == 0:
                freqs = pr.exact_freqs(sh, self.pstart, lists, offsets, cand)
            else:
                idx = [p[np.searchsorted(d, cand)] for p, d in lists]
                pos = lambda p: sh.post_positions[self.pstart[p]:self.pstart[p + 1]].tolist()   # noqa: E731
                freqs = np.array([pr.sloppy_freq([pos(idx[i][k]) for i in range(len(terms))], offsets, q.slop)
                                  for k in range(len(cand))], np.float32)
            docs, freqs = cand[freqs > 0], freqs[freqs > 0]
            present[docs] = True
            score[docs] = bm25(w, freqs, self.norms(f, docs), self.caches[f])
        return present, score

    # ------------------------------------------------------------ nodes

    def eval(self, q, boost=F32(1)):
        """(present, score) of query object q under the folded boost `boost`"""
        q, boost = fold_boost(q, boost)
        if isinstance(q, BooleanQuery):
            return self.boolean(q, boost)
        if isinstance(q, DisjunctionMaxQuery):
            return self.dismax(q, boost)
        key = (repr(q), boost.tobytes())   # leaves only: a node's arrays are not kept
        if key in self.memo:
            return self.memo[key]
        if isinstance(q, TermQuery):
            out = self.term(int(q.term), boost)
        elif isinstance(q, PhraseQuery):
            out = self.phrase(q, boost)
        elif isinstance(q, (RangeQuery, KeywordRangeQuery, KeywordPrefixQuery, MatchAllDocsQuery)):
            p = (self.range_(q) if isinstance(q, RangeQuery) else np.ones(self.n, bool) if isinstance(q, MatchAllDocsQuery)
                 else self.keyword(q))
            out = p, np.where(p, boost, F32(0)).astype(np.float32)
        else:
            raise TypeError(f"no reference for {type(q).__name__}")
        if len(self.memo) >= self.max_memo:
            self.memo.clear()
        self.memo[key] = out
        return out

    def boolean(self, q: BooleanQuery, boost):
        n = self.n
        ok = np.ones(n, bool)
        must, should = np.zeros(n, np.float64), np.zeros(n, np.float64)
        n_should = np.zeros(n, np.int32)
        n_req = 0
        for c in q.clauses:
            p, s = self.eval(c.query, boost)
            if c.occur in (Occur.MUST, Occur.FILTER):
                n_req += 1
                ok &= p
            elif c.occur == Occur.MUST_NOT:
                ok &= ~p
            else:
                n_should += p
                should = np.where(p, should + s.astype(np.float64), should)
            if c.occur == Occur.MUST:
                must = np.where(p, must + s.astype(np.float64), must)
        msm = q.minimum_number_should_match
        ok &= n_should >= (msm if msm > 0 else (1 if n_req == 0 else 0))
        if n_req == 0:
            score = should.astype(np.float32)
        else:
            req, opt = must.astype(np.float32), should.astype(np.float32)
            both = (req.astype(np.float64) + opt.astype(np.float64)).astype(np.float32) if msm > 0 else req + opt
            score = np.where(n_should > 0, both, req)
        return ok, np.where(ok, score, F32(0)).astype(np.float32)

    def dismax(self, q: DisjunctionMaxQuery, boost):
        n = self.n
        mx, others = np.zeros(n, np.float32), np.zeros(n, np.float64)
        any_ = np.zeros(n, bool)
        for d in q.disjuncts:
            p, s = self.eval(d, boost)
            new_max = p & (s >= mx)
            others = np.where(new_max, others + mx.astype(np.float64), np.where(p, others + s.astype(np.float64), others))
            mx = np.where(new_max, s, mx)
            any_ |= p
        score = (mx.astype(np.float64) + others * np.float64(F32(q.tie_breaker))).astype(np.float32)
        return any_, np.where(any_, score, F32(0)).astype(np.float32)

    # ------------------------------------------------------------ pages

    def matches(self, q):
        """(live matches: local doc ids ascending, their float32 scores)"""
        p, s = self.eval(q)
        m = np.nonzero(p & self.live)[0]
        return m, s[m]

    def page(self, q, top_k: int, after=None):
        """(global docs, scores, total hits) of one query's page; after: a ScoreDoc (global doc) or None"""
        m, sc = self.matches(q)
        return self.page_of(m, sc, top_k, after)

    def page_of(self, m, sc, top_k: int, after=None):
        """page() of the live matches m (local ids) with scores sc"""
        gdoc = m.astype(np.int64) + self.sh.doc_base
        total = len(m)
        if after is not None:
            a = F32(after.score)
            keep = (sc < a) | ((sc == a) & (gdoc > after.doc))
            sc, gdoc = sc[keep], gdoc[keep]
        order = np.lexsort((gdoc, -sc.astype(np.float64)))[:top_k]
        return gdoc[order].astype(np.int32), sc[order], total

    def search(self, queries, top_k: int, search_after=None):
        """docs [nq, k], scores [nq, k], counts [nq], total hits [nq] (exact), as the engines return them"""
        nq = len(queries)
        docs, scores = np.zeros((nq, top_k), np.int32), np.zeros((nq, top_k), np.float32)
        counts, total = np.zeros(nq, np.int32), np.zeros(nq, np.int64)
        for i, q in enumerate(queries):
            d, s, t = self.page(q, top_k, None if search_after is None else search_after[i])
            docs[i, :len(d)], scores[i, :len(d)], counts[i], total[i] = d, s, len(d), t
        return docs, scores, counts, total


def _bytes(v) -> bytes:
    return v.encode("utf-8") if isinstance(v, str) else bytes(v)
