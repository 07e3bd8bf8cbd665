#!/usr/bin/env python
"""QueryRescorer with a tree or phrase rescore query (nrtgpu_rescore_query_tree) on tools/phrase_bench.py's 10M-doc
two-field shard with positions (its generators; a bag-of-terms body field 0 and a title-like field 1 with bigrams).
Batches of 1024 queries; each query is 2-3 consecutive title tokens of a random doc:
  (1) first pass match(tokens) top 1000, rescored by the exact phrase of the tokens at window 1000;
  (2) the same rescored by the phrase at slop 2;
  (3) the exact phrase at window 100 (top 1000), and at window 4096 (the first pass paged by searchAfter to 4096 hits);
  (4) a multi_match rescore query without phrases: DisjunctionMaxQuery(match(tokens), match(two body terms)), tie 0.3.
Weights (1, 4) as in QueryTest. Each workload first checks an 8-query sample of the rescored pages, bit-exact, against
tests/rescore_tree_reference.py and oracle.rescore_combine; a failed check stops the run. Prints one JSON line per workload:
the whole nrtgpu_rescore_query_tree call by host clock (hit lists and scores from the host and the rescored page back on
the host), the device span of the call by CUDA events on its stream (uploads, both kernels, the copies back), and the
device time of score_docs_tree_kernel from torch.profiler in a separate pass, with the card name and power limit read in the
same run.
python tools/rescore_bench.py [--docs 10000000] [--nq 1024] [--steps 10] [--warmup 2] [--sample 8]"""
import argparse, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # the references
sys.path.insert(0, os.path.join(ROOT, "tools"))
from phrase_bench import field0_positions, field1_tokens   # noqa: E402
from tree_bench import card   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000); ap.add_argument("--vocab1", type=int, default=100_000)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=8, help="queries per workload checked against the reference")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build_if_needed()
    import torch
    import oracle
    import phrase_reference as pref
    import rescore_tree_reference as rr
    from nrtsearch_b200 import index as ix
    from nrtsearch_b200.search import (BooleanQuery, DisjunctionMaxQuery, GpuContext, GpuIndex, GpuIndexSearcher, Occur, PhraseQuery,
                                       RelevanceCollector, ScoreDoc, TermQuery)
    n, nq = a.docs, a.nq
    # the corpus of tools/phrase_bench.py, built the same way from its generators and seeds
    rng = np.random.default_rng(17)
    f0 = ix.synth_text_shard(n, a.vocab)
    lut = np.array([oracle.byte4_to_int(b) for b in range(256)], np.int64)
    pos0 = field0_positions(f0, lut[f0.fields[0].norms])
    doc1, tok1, p1, start1 = field1_tokens(n, a.vocab1, rng)
    f1 = pref.shard_from_token_arrays(n, np.zeros(a.vocab1, np.int32), 1, doc1, tok1, p1)
    sh = ix.HostShard(n_docs=n, doc_base=0, term_off=np.concatenate([f0.term_off, f0.term_off[-1] + f1.term_off[1:]]),
                      post_docs=np.concatenate([f0.post_docs, f1.post_docs]), post_freqs=np.concatenate([f0.post_freqs, f1.post_freqs]),
                      fields=[f0.fields[0], f1.fields[0]],
                      term_field=np.concatenate([np.zeros(a.vocab, np.int32), np.ones(a.vocab1, np.int32)]),
                      post_positions=np.concatenate([pos0, f1.post_positions]))
    sh.term_df = np.diff(sh.term_off).astype(np.int64)
    del f0, f1, pos0
    sh.columns, sh.column_has = [ix.synth_int_column(n)], [None]
    phrases = []   # 2-3 consecutive title tokens of random docs, without a repeated token
    while len(phrases) < nq:
        d = int(rng.integers(0, n))
        L = int(min(start1[d + 1] - start1[d], rng.integers(2, 4)))
        s = int(rng.integers(0, start1[d + 1] - start1[d] - L + 1))
        p = [int(t) + a.vocab for t in tok1[start1[d] + s:start1[d] + s + L]]
        if len(set(p)) == len(p):
            phrases.append(p)
    body = ix.synth_query_terms(nq, 2, a.vocab)

    def match(ts):
        q = BooleanQuery()
        for t in ts:
            q.add(TermQuery(int(t)), Occur.SHOULD)
        return q

    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    first = [match(p) for p in phrases]
    page = s.search_tree(first, RelevanceCollector(1000, 1000))
    # window 4096: the first pass paged to 4096 hits by searchAfter (top_k is at most 1024 per page)
    docs4 = np.zeros((nq, 4096), np.int32); scores4 = np.zeros((nq, 4096), np.float32); counts4 = np.zeros(nq, np.int32)
    after = None
    for pg in range(4):
        r = s.search_tree(first, RelevanceCollector(1024, 1000), search_after=after)
        for q in range(nq):
            c = int(r.counts[q])
            docs4[q, counts4[q]:counts4[q] + c] = r.docs[q, :c]; scores4[q, counts4[q]:counts4[q] + c] = r.scores[q, :c]
            counts4[q] += c
        after = [ScoreDoc(int(docs4[q, counts4[q] - 1]), float(scores4[q, counts4[q] - 1])) if counts4[q] else None for q in range(nq)]
    exact = [PhraseQuery(p) for p in phrases]
    hits1000 = (page.docs, page.scores, page.counts)
    workloads = [
        ("(1) match top 1000 -> exact phrase, window 1000", exact, hits1000, 1000),
        ("(2) match top 1000 -> phrase slop 2, window 1000", [PhraseQuery(p, slop=2) for p in phrases], hits1000, 1000),
        ("(3a) match top 1000 -> exact phrase, window 100", exact, hits1000, 100),
        ("(3b) match top 4096 -> exact phrase, window 4096", exact, (docs4, scores4, counts4), 4096),
        ("(4) match top 1000 -> multi_match dismax (no phrase), window 1000",
         [DisjunctionMaxQuery([match(p), match(b)], 0.3) for p, b in zip(phrases, body)], hits1000, 1000),
    ]
    base = {"docs": n, "fields": 2, "batch": nq, "weights": [1.0, 4.0], "gpu": card()}
    oix = oracle.OracleIndex(sh)
    leaves = pref.PhraseLeaves(sh, oix, None, None)
    sample = list(range(0, nq, max(1, nq // a.sample)))[:a.sample]
    stream = torch.cuda.Stream()
    for name, queries, (d0, s0, c0), window in workloads:
        run = lambda: s.rescore_query_tree(queries, d0, s0, c0, window, 1.0, 4.0, stream=stream.cuda_stream)  # noqa: E731
        d, sc, c = run()
        m, s2 = rr.score_docs(sh, [queries[q] for q in sample], d0[sample], c0[sample], oix=oix, leaves=leaves)
        wd, ws, wc = rr.rescore(d0[sample], s0[sample], m, s2, c0[sample], window, 1.0, 4.0)
        for i, q in enumerate(sample):
            k = int(wc[i])
            if not (c[q] == k and np.array_equal(d[q, :k], wd[i, :k]) and np.array_equal(sc[q, :k].view(np.uint32), ws[i, :k].view(np.uint32))):
                raise SystemExit(f"{name}: GPU rescore differs from the reference (query {q})")
        for _ in range(a.warmup):
            run()
        host, dev = [], []
        for _ in range(a.steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t = time.perf_counter()
            e0.record(stream)
            run()   # returns after the rescored page is on the host (the call synchronises its stream)
            e1.record(stream)
            host.append(time.perf_counter() - t)
            e1.synchronize()
            dev.append(e0.elapsed_time(e1))
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                run()
        kern = {}
        for ev in prof.key_averages():
            if "score_docs_tree_kernel" in ev.key or "rescore_combine_kernel" in ev.key:
                kern["score_docs_tree_kernel" if "score_docs" in ev.key else "rescore_combine_kernel"] = \
                    round(ev.device_time_total / 1e3 / ev.count, 3)
        med = float(np.median(host))
        print(json.dumps({**base, "workload": name, "window": window, "hits": int(c0.sum()), "call_ms_median": round(1e3 * med, 3),
                          "call_ms_min": round(1e3 * min(host), 3), "call_device_ms_median": round(float(np.median(dev)), 3),
                          "kernel_ms": kern, "sample_second_pass_matches": int(m.sum()), "steps": a.steps,
                          "reference_gate": f"{len(sample)} queries bit-exact"}), flush=True)
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
