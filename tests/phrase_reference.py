"""Reference for phrase leaves of query trees (PhraseQuery, nrtgpu_search_tree_phrases), the checker of the window engine's
phrase matching. TEST INFRASTRUCTURE ONLY.

  - exact_freq / sloppy_freq restate Lucene 10's ExactPhraseMatcher and SloppyPhraseMatcher (without repeats) step by step
    on one doc's positions; exact_freqs counts the same thing for many docs at once (a lead position matches when every
    other term holds the position it implies), and the tests pin the two against each other;
  - PhraseLeaves extends tree_reference.LeafScores with phrase leaves: freq over every doc that holds all the terms, weight
    boost * (float) of the double sum of the terms' idf (oracle.bm25_idf), score through oracle's orc_bm25_score;
  - search_tree combines them with tree_reference's node rules (tree_reference.evaluate takes the leaf callable);
  - shard_from_tokens / shard_from_token_arrays build a shard with positions from token sequences, multi-valued fields
    separated by a position increment gap (the adaptor's: TextBaseFieldDef, default 100)."""
import ctypes as C

import numpy as np

import oracle
import tree_reference as tr
from nrtsearch_b200 import _native
from nrtsearch_b200 import index as ix

PHRASE = 4
GAP = 100


# ---------------------------------------------------------------- the matchers on one doc

def exact_freq(term_positions, offsets, first_only=False) -> np.float32:
    """ExactPhraseMatcher: term_positions[i] are term i's positions in the doc (ascending), offsets[i] its query position,
    the terms ordered by query position (term 0 leads). Sum of sloppyWeight (1) over the matches."""
    n = len(term_positions)
    pos, upto = [-1] * n, [0] * n

    def advance(i, target):   # advancePosition
        while pos[i] < target:
            if upto[i] == len(term_positions[i]):
                return False
            pos[i] = term_positions[i][upto[i]]
            upto[i] += 1
        return True

    freq = np.float32(0)
    while upto[0] < len(term_positions[0]):   # nextMatch
        pos[0] = term_positions[0][upto[0]]
        upto[0] += 1
        matched = False
        while True:   # advanceHead
            phrase_pos = pos[0] - offsets[0]
            again = failed = False
            for j in range(1, n):
                expected = phrase_pos + offsets[j]
                if not advance(j, expected):
                    failed = True
                    break
                if pos[j] != expected:   # advanced too far: move the lead
                    if advance(0, pos[j] - offsets[j] + offsets[0]):
                        again = True
                    else:
                        failed = True
                    break
            if failed or not again:
                matched = not failed
                break
        if not matched:
            break
        freq = np.float32(freq + np.float32(1))
        if first_only:
            break
    return freq


def sloppy_freq(term_positions, offsets, slop, first_only=False) -> np.float32:
    """SloppyPhraseMatcher without repeated terms: PhraseQueue ordered by (position - offset, offset, ordinal), the running
    end, the match-length minimisation; each match adds 1.0f / (1.0f + matchLength) in float."""
    n = len(term_positions)
    pos, cnt = [0] * n, [0] * n
    end = -(2**31)
    for i in range(n):
        pos[i] = term_positions[i][0] - offsets[i]
        cnt[i] = 1
        end = max(end, pos[i])
    queue = set(range(n))
    key = lambda i: (pos[i], offsets[i], i)   # noqa: E731

    def pop():
        i = min(queue, key=key)
        queue.remove(i)
        return i

    freq = np.float32(0)
    positioned = True
    while positioned:   # nextMatch
        pp = pop()
        match_length = end - pos[pp]
        nxt = pos[min(queue, key=key)]
        while True:
            if cnt[pp] == len(term_positions[pp]):   # pp exhausted
                positioned = False
                matched = match_length <= slop
                break
            pos[pp] = term_positions[pp][cnt[pp]] - offsets[pp]
            cnt[pp] += 1
            end = max(end, pos[pp])
            if pos[pp] > nxt:   # done minimising the current match length
                queue.add(pp)
                if match_length <= slop:
                    matched = True
                    break
                pp = pop()
                nxt = pos[min(queue, key=key)]
                match_length = end - pos[pp]
            else:
                match_length = min(match_length, end - pos[pp])
        if not matched:
            break
        freq = np.float32(freq + np.float32(1) / (np.float32(1) + np.float32(match_length)))
        if first_only:
            break
    return freq


def phrase_freq(term_positions, offsets, slop, first_only=False) -> np.float32:
    return exact_freq(term_positions, offsets, first_only) if slop == 0 else sloppy_freq(term_positions, offsets, slop, first_only)


# ---------------------------------------------------------------- phrase leaves over a shard

class PhraseLeaves(tr.LeafScores):
    """tree_reference.LeafScores plus phrase leaves (clause kind 4) of the phrase table parr / tarr"""

    def __init__(self, sh, oix, parr, tarr):
        super().__init__(sh, oix)
        self.parr, self.tarr = parr, tarr
        self.pstart = np.zeros(len(sh.post_freqs) + 1, np.int64)
        np.cumsum(sh.post_freqs, out=self.pstart[1:])

    def term_postings(self, t):
        a, b = int(self.sh.term_off[t]), int(self.sh.term_off[t + 1])
        return np.arange(a, b), self.sh.post_docs[a:b]

    def positions(self, p):
        return self.sh.post_positions[self.pstart[p]:self.pstart[p + 1]].tolist()

    def __call__(self, c):
        if c.kind != PHRASE:
            return super().__call__(c)
        ph = self.parr[c.id]
        terms = [(int(self.tarr[i].term), int(self.tarr[i].position)) for i in range(ph.term_begin, ph.term_end)]
        n = self.sh.n_docs
        if not terms:   # MatchNoDocsQuery
            return np.zeros(n, bool), np.zeros(n, np.float32)
        if len(terms) == 1:   # rewritten to the TermQuery
            return super().__call__(_native.Clause(c.occur, 0, terms[0][0], c.boost, 0, 0))
        key = ("phrase", tuple(terms), int(ph.slop), np.float32(c.boost).tobytes(), c.occur in (tr.FILTER, tr.MUST_NOT))
        if key in self.cache:
            return self.cache[key]
        terms = sorted(terms, key=lambda t: t[1])   # stable: the lead is the first of the smallest position
        sh = self.sh
        f = int(sh.term_field[terms[0][0]]) if sh.term_field is not None else 0
        fld = sh.fields[f]
        df = sh.term_df if sh.term_df is not None else np.diff(sh.term_off)
        idf = 0.0
        for t, _ in terms:
            idf += float(oracle.bm25_idf(max(int(df[t]), 1), fld.doc_count))
        weight = np.float32(np.float32(c.boost) * np.float32(idf))
        lists = [self.term_postings(t) for t, _ in terms]
        cand = lists[0][1]
        for _, d in lists[1:]:
            cand = np.intersect1d(cand, d, assume_unique=True)
        offsets = [p for _, p in terms]
        present, score = np.zeros(n, bool), np.zeros(n, np.float32)
        if len(cand):
            if ph.slop == 0:
                freqs = exact_freqs(sh, self.pstart, lists, offsets, cand)
            else:
                idx = [p[np.searchsorted(d, cand)] for p, d in lists]
                freqs = np.array([sloppy_freq([self.positions(idx[i][k]) for i in range(len(terms))], offsets, ph.slop)
                                  for k in range(len(cand))], np.float32)
            hit = freqs > 0
            docs, freqs = cand[hit], freqs[hit]
            present[docs] = True
            cache = oracle.bm25_cache(fld.k1, fld.b, float(oracle.lib().orc_bm25_avgdl(fld.sum_total_term_freq, fld.doc_count)))
            cp = cache.ctypes.data_as(C.POINTER(C.c_float))
            for d, fr in zip(docs.tolist(), freqs.tolist()):
                nb = int(fld.norms[d]) if fld.norms is not None else 1
                score[d] = oracle.lib().orc_bm25_score(weight, fr, nb, cp)
        self.cache[key] = (present, score)
        return present, score


def exact_freqs(sh, pstart, lists, offsets, cand) -> np.ndarray:
    """exact_freq of every doc of cand at once: the lead's positions (each occurrence) at which every other term holds
    lead - offsets[0] + offsets[j], counted per doc (float32 [len(cand)])"""
    def entries(j):
        p, d = lists[j]
        sel = p[np.isin(d, cand)]
        f = (pstart[sel + 1] - pstart[sel])
        docs = np.repeat(sh.post_docs[sel].astype(np.int64), f)
        pos = sh.post_positions[np.repeat(pstart[sel] - (np.cumsum(f) - f), f) + np.arange(int(f.sum()))].astype(np.int64)
        return docs, pos
    ld, lp = entries(0)
    ok = np.ones(len(ld), bool)
    for j in range(1, len(lists)):
        d, p = entries(j)
        ok &= np.isin(ld * (1 << 33) + (lp - offsets[0] + offsets[j]), d * (1 << 33) + p)
    counts = np.bincount(np.searchsorted(cand, ld[ok]), minlength=len(cand))
    return counts.astype(np.float32)


def search_tree(sh, carr, ncl, narr, nn, parr, n_ph, tarr, n_pt, qarr, nq, top_k, oix=None, leaves=None):
    """docs [nq, k] (global), scores [nq, k], counts [nq], total hits [nq] (exact), relation [nq] (0): tree_reference's
    search_tree with phrase leaves"""
    oix = oix or oracle.OracleIndex(sh)
    leaves = leaves or PhraseLeaves(sh, oix, parr, tarr)
    docs = np.zeros((nq, top_k), np.int32)
    scores = np.zeros((nq, top_k), np.float32)
    counts = np.zeros(nq, np.int32)
    total = np.zeros(nq, np.int64)
    for q in range(nq):
        qq = qarr[q]
        p, s = tr.evaluate(sh, carr, narr, qq.clause_begin, qq.clause_end, qq.min_should_match, leaves)
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


def search(sh, queries, top_k, search_after=None, oix=None, leaves=None):
    """search_tree over nrtsearch_b200.search query objects (PhraseQuery leaves included)"""
    from nrtsearch_b200.search import compile_tree
    a = compile_tree(queries, search_after, phrase_table=True)
    return search_tree(sh, *a, top_k, oix, leaves)


# ---------------------------------------------------------------- shards with positions

def shard_from_token_arrays(n_docs, term_field, n_fields, doc, term, pos, live_docs=None) -> ix.HostShard:
    """A shard from flat token arrays (doc, term, position): postings in CSR order with freqs and positions, norms from the
    field lengths (every token counts), docCount / sumTotalTermFreq per field, term_df = list lengths."""
    term_field = np.asarray(term_field, np.int32)
    doc, term, pos = (np.asarray(a, np.int64) for a in (doc, term, pos))
    order = np.lexsort((pos, doc, term))
    doc, term, pos = doc[order], term[order], pos[order]
    new = np.ones(len(doc), bool)
    new[1:] = (term[1:] != term[:-1]) | (doc[1:] != doc[:-1])
    starts = np.nonzero(new)[0]
    freqs = np.diff(np.append(starts, len(doc))).astype(np.int32)
    pterm = term[starts]
    term_off = np.zeros(len(term_field) + 1, np.int64)
    np.cumsum(np.bincount(pterm, minlength=len(term_field)), out=term_off[1:])
    fields = []
    tf = term_field[term]
    for f in range(n_fields):
        lens = np.bincount(doc[tf == f], minlength=n_docs)
        table = np.array([oracle.int_to_byte4(int(x)) for x in range(int(lens.max()) + 1)], np.uint8)
        fields.append(ix.TextField(table[lens], int((lens > 0).sum()), int(lens.sum())))
    return ix.HostShard(n_docs=n_docs, doc_base=0, term_off=term_off, post_docs=doc[starts].astype(np.int32), post_freqs=freqs,
                        fields=fields, term_field=term_field, term_df=np.diff(term_off).astype(np.int64),
                        live_docs=live_docs, post_positions=pos.astype(np.int32))


def shard_from_tokens(docs, term_field, n_fields, gap=GAP) -> ix.HostShard:
    """docs[d][f] = the values of text field f in doc d, each a list of term ids; the first token of a value takes the
    position after the previous value's last one plus gap (Lucene's position increment gap between values)"""
    d_, t_, p_ = [], [], []
    for d, doc in enumerate(docs):
        for values in doc:
            p = -1
            for k, v in enumerate(values):
                if k > 0:
                    p += gap
                for t in v:
                    p += 1
                    d_.append(d), t_.append(t), p_.append(p)
    return shard_from_token_arrays(len(docs), term_field, n_fields, d_, t_, p_)
