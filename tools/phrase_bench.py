#!/usr/bin/env python
"""Phrase queries (nrtgpu_search_tree_phrases) on tools/tree_bench.py's 10M-doc two-field shard, with positions:
  field 0  the bench corpus (1M-term vocabulary, mean length 56) as synth_text_shard makes it, a bag of terms: every posting
           takes positions at a hashed offset inside the doc's length, so that phrases occur about as often as chance makes
           them (a random position order per doc);
  field 1  a short title-like field (100K terms, 2 + Poisson(6) tokens) generated as token sequences in which half the
           tokens follow their predecessor by a fixed map, so that bigram phrases occur.
Batches of 1024 queries, top 100, totalHitsThreshold 1000, phrases of 2-3 consecutive field-1 tokens of random docs:
  (a) match_phrase on field 1;  (b) the same phrases at slop 2;  (c) MUST match(tokens) + SHOULD phrase(tokens)^2 on field 1;
  (d) match_phrase of two log-uniform field-0 terms.
Every workload is first checked on a sample of queries, bit-exact on docs, scores, counts and totalHits, against
tests/phrase_reference.py; a failed check stops the run. Prints one JSON line per workload with the batch time (host clock
around a call that ends with the results on the host), the search kernel time (CUDA events of a prepared batch), the device
bytes of the positions, and the card name and power limit read in the same run.
python tools/phrase_bench.py [--docs 10000000] [--nq 1024] [--k 100] [--steps 10] [--warmup 2] [--sample 8]"""
import argparse, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # phrase_reference: the checker of the phrases
sys.path.insert(0, os.path.join(ROOT, "tools"))
from tree_bench import card   # noqa: E402


def field0_positions(sh, lengths):
    """positions of every posting of the bag-of-terms field 0: posting (t, d) of freq f at h(t, d) mod len(d) + 0..f-1"""
    out = np.empty(int(sh.post_freqs.sum()), np.int32)
    pstart = np.zeros(len(sh.post_freqs) + 1, np.int64)
    np.cumsum(sh.post_freqs, out=pstart[1:])
    terms = np.repeat(np.arange(sh.n_terms, dtype=np.int64), np.diff(sh.term_off))
    step = 1 << 24
    for a in range(0, len(sh.post_docs), step):
        b = min(a + step, len(sh.post_docs))
        d = sh.post_docs[a:b].astype(np.int64)
        f = sh.post_freqs[a:b].astype(np.int64)
        h = ((terms[a:b] * 0x9E3779B1 + d * 0x85EBCA77) >> 7) % np.maximum(lengths[d], 1)
        first = np.repeat(h - (np.cumsum(f) - f), f)
        out[pstart[a]:pstart[b]] = first + np.arange(int(f.sum()))
    return out


def field1_tokens(n, vocab, rng):
    lens = 2 + rng.poisson(6.0, n)
    start = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=start[1:])
    w = 1.0 / np.arange(1, vocab + 1)
    tok = np.searchsorted(np.cumsum(w) / w.sum(), rng.random(int(start[-1]))).astype(np.int64)
    doc = np.repeat(np.arange(n), lens)
    pos = np.arange(int(start[-1])) - start[doc]
    follow = (rng.random(len(tok)) < 0.5) & (pos > 0)
    for _ in range(3):   # a followed token is a fixed function of its predecessor (a bigram model of order 1, in three passes)
        idx = np.nonzero(follow)[0]
        tok[idx] = (tok[idx - 1] * 7919 + 13) % vocab
    return doc, tok, pos, start


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000); ap.add_argument("--vocab1", type=int, default=100_000)
    ap.add_argument("--nq", type=int, default=1024); ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=8, help="queries per workload checked against the reference")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build_if_needed()
    import oracle
    import phrase_reference as ref
    from nrtsearch_b200 import index as ix
    from nrtsearch_b200.search import (BooleanQuery, BoostQuery, GpuContext, GpuIndex, GpuIndexSearcher, Occur, PhraseQuery,
                                       RelevanceCollector, TermQuery)
    n, nq, k = a.docs, a.nq, a.k
    rng = np.random.default_rng(17)
    f0 = ix.synth_text_shard(n, a.vocab)
    lut = np.array([oracle.byte4_to_int(b) for b in range(256)], np.int64)
    pos0 = field0_positions(f0, lut[f0.fields[0].norms])
    doc1, tok1, p1, start1 = field1_tokens(n, a.vocab1, rng)
    f1 = ref.shard_from_token_arrays(n, np.zeros(a.vocab1, np.int32), 1, doc1, tok1, p1)
    sh = ix.HostShard(n_docs=n, doc_base=0, term_off=np.concatenate([f0.term_off, f0.term_off[-1] + f1.term_off[1:]]),
                      post_docs=np.concatenate([f0.post_docs, f1.post_docs]), post_freqs=np.concatenate([f0.post_freqs, f1.post_freqs]),
                      fields=[f0.fields[0], f1.fields[0]],
                      term_field=np.concatenate([np.zeros(a.vocab, np.int32), np.ones(a.vocab1, np.int32)]),
                      post_positions=np.concatenate([pos0, f1.post_positions]))
    sh.term_df = np.diff(sh.term_off).astype(np.int64)
    del f0, f1, pos0
    sh.columns, sh.column_has = [ix.synth_int_column(n)], [None]
    # phrases: 2-3 consecutive field-1 tokens of random docs
    phrases = []   # (without a repeated token: a sloppy phrase with one is not on the GPU path)
    while len(phrases) < nq:
        d = int(rng.integers(0, n))
        L = int(min(start1[d + 1] - start1[d], rng.integers(2, 4)))
        s = int(rng.integers(0, start1[d + 1] - start1[d] - L + 1))
        p = [int(t) + a.vocab for t in tok1[start1[d] + s:start1[d] + s + L]]
        if len(set(p)) == len(p):
            phrases.append(p)
    t0 = ix.synth_query_terms(nq, 2, a.vocab)

    def match(ts):
        q = BooleanQuery()
        for t in ts:
            q.add(TermQuery(t), Occur.SHOULD)
        return q

    workloads = [
        ("(a) match_phrase, field 1", [PhraseQuery(p) for p in phrases]),
        ("(b) match_phrase slop 2, field 1", [PhraseQuery(p, slop=2) for p in phrases]),
        ("(c) MUST match + SHOULD phrase^2, field 1",
         [BooleanQuery().add(match(p), Occur.MUST).add(BoostQuery(PhraseQuery(p), 2.0), Occur.SHOULD) for p in phrases]),
        ("(d) match_phrase, field 0", [PhraseQuery([int(x[0]), int(x[1])]) for x in t0]),
    ]
    ctx = GpuContext(0)
    positions = sh.post_positions
    sh.post_positions = None
    gix = GpuIndex(ctx, sh)
    before = gix.device_bytes
    gix.add_positions(positions)
    sh.post_positions = positions
    pos_bytes = gix.device_bytes - before
    s = GpuIndexSearcher(gix)
    base = {"docs": n, "fields": 2, "batch": nq, "top_k": k, "threshold": 1000, "positions": int(len(positions)),
            "positions_device_bytes": int(pos_bytes), "image_device_bytes": int(gix.device_bytes), "gpu": card()}
    oix = oracle.OracleIndex(sh)
    sample = list(range(0, nq, max(1, nq // a.sample)))[:a.sample]
    col = RelevanceCollector(k, 1000)

    def gate(name, res, queries):
        wd, ws, wc, wt, _ = ref.search(sh, [queries[i] for i in sample], k, oix=oix)
        for i, q in enumerate(sample):
            c = wc[i]
            if not (res.counts[q] == c and np.array_equal(res.docs[q, :c], wd[i, :c])
                    and np.array_equal(res.scores[q, :c].view(np.uint32), ws[i, :c].view(np.uint32)) and res.total_hits[q] == wt[i]):
                raise SystemExit(f"{name}: GPU results differ from the reference (query {q})")

    def timed(run):
        for _ in range(a.warmup):
            run()
        ts = []
        for _ in range(a.steps):
            t = time.perf_counter()
            run()   # every call copies its results to the host and synchronises
            ts.append(time.perf_counter() - t)
        return ts

    for name, queries in workloads:
        run = lambda q=queries: s.search_tree(q, col)   # noqa: E731
        res = run()
        gate(name, res, queries)
        ts = timed(run)
        b = s.prepare_tree(queries, col)
        for _ in range(a.warmup):
            b.run(); b.fetch()
        b.reset_timing()
        for _ in range(a.steps):
            b.run(); b.fetch()
        kms, items = b.stage_ms(0), b.stats()["work_items"]
        b.close()
        med = float(np.median(ts))
        print(json.dumps({**base, "workload": name, "ms_median": round(1e3 * med, 3), "ms_min": round(1e3 * min(ts), 3),
                          "qps": round(nq / med, 1), "kernel_ms": round(kms, 3), "work_items": items, "steps": a.steps,
                          "matching_queries": int((res.total_hits > 0).sum()),
                          "oracle_gate": f"{len(sample)} queries bit-exact"}), flush=True)
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
