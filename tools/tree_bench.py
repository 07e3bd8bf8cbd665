#!/usr/bin/env python
"""Query trees (nrtgpu_search_tree) on a 10M-doc synthetic shard with two text fields -- field 0 the bench corpus (1M-term
vocabulary, mean length 56), field 1 a short title-like field (100K terms, mean length 8) -- and the bench's price column.
Batches of 1024 queries, top 100, totalHitsThreshold 1000. Three workloads:
  (a) match-in-bool + range: BooleanQuery(MUST BooleanQuery(SHOULD t1, SHOULD t2), FILTER price range), search_tree;
  (b) the same queries flattened, BooleanQuery(SHOULD t1, SHOULD t2, FILTER range, msm 1), search_batch (the probe path);
      it matches the same docs with the same scores;
  (c) multi_match BEST_FIELDS over both fields + range, BooleanQuery(MUST DisjunctionMaxQuery([match on field 0, match on
      field 1], tie), FILTER range), at tie_breaker 0 and 0.3, search_tree.
Every workload is first checked on a sample of queries, bit-exact on docs, scores, counts and totalHits, against
tests/tree_reference.py (trees) or the oracle (flat); a failed check stops the run. Prints one JSON line per workload with
the batch time (host clock around a call that ends with the results on the host), the search kernel time (CUDA events of a
prepared batch), and the card name and power limit read in the same run.
python tools/tree_bench.py [--docs 10000000] [--nq 1024] [--k 100] [--steps 10] [--warmup 2] [--sample 8]"""
import argparse, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # tree_reference: the checker of the trees


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the JSON still says what was measured on
        return f"unknown ({e})"


def two_field_shard(n, vocab0, vocab1):
    from nrtsearch_b200 import index as ix
    a = ix.synth_text_shard(n, vocab0)
    b = ix.synth_text_shard(n, vocab1, seed=ix.SEED_CORPUS + 7, min_len=2, poisson_mean=6.0)
    sh = ix.HostShard(n_docs=n, doc_base=0, term_off=np.concatenate([a.term_off, a.term_off[-1] + b.term_off[1:]]),
                      post_docs=np.concatenate([a.post_docs, b.post_docs]), post_freqs=np.concatenate([a.post_freqs, b.post_freqs]),
                      fields=[a.fields[0], b.fields[0]],
                      term_field=np.concatenate([np.zeros(vocab0, np.int32), np.ones(vocab1, np.int32)]))
    sh.columns = [ix.synth_int_column(n)]
    sh.column_has = [None]
    return sh


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
    import tree_reference as ref
    from nrtsearch_b200 import index as ix
    from nrtsearch_b200.search import (BooleanQuery, DisjunctionMaxQuery, GpuContext, GpuIndex, GpuIndexSearcher, Occur, RangeQuery,
                                       RelevanceCollector, TermQuery, compile_queries)
    n, nq, k = a.docs, a.nq, a.k
    sh = two_field_shard(n, a.vocab, a.vocab1)
    t = ix.synth_query_terms(nq, 2, a.vocab)
    u = ix.synth_query_terms(nq, 2, a.vocab1, seed=ix.SEED_QUERIES + 1) + a.vocab
    price = RangeQuery(0, 100_000, 600_000)

    def match(x):
        return BooleanQuery().add(TermQuery(int(x[0])), Occur.SHOULD).add(TermQuery(int(x[1])), Occur.SHOULD)

    tree = [BooleanQuery().add(match(x), Occur.MUST).add(price, Occur.FILTER) for x in t]
    flat = [BooleanQuery(minimum_number_should_match=1).add(TermQuery(int(x[0])), Occur.SHOULD).add(TermQuery(int(x[1])), Occur.SHOULD)
            .add(price, Occur.FILTER) for x in t]

    def multi(tie):
        return [BooleanQuery().add(DisjunctionMaxQuery([match(x), match(y)], tie), Occur.MUST).add(price, Occur.FILTER)
                for x, y in zip(t, u)]

    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    gpu = card()
    base = {"docs": n, "fields": 2, "batch": nq, "top_k": k, "threshold": 1000, "gpu": gpu}
    oix = oracle.OracleIndex(sh)
    sample = list(range(0, nq, max(1, nq // a.sample)))[:a.sample]
    col = RelevanceCollector(k, 1000)

    def gate(name, res, queries, is_tree):
        sub = [queries[i] for i in sample]
        if is_tree:
            wd, ws, wc, wt, _ = ref.search(sh, sub, k, oix=oix)
        else:
            carr, ncl, qarr, snq = compile_queries(sub)
            wd, ws, wc, wt, _ = oracle.search_compiled(oix, carr, ncl, qarr, snq, k, n_threads=8)
        for i, q in enumerate(sample):
            c = wc[i]
            exact_total = res.relation[q] == 0
            if not (res.counts[q] == c and np.array_equal(res.docs[q, :c], wd[i, :c])
                    and np.array_equal(res.scores[q, :c].view(np.uint32), ws[i, :c].view(np.uint32))
                    and (res.total_hits[q] == wt[i] if exact_total else 1000 < res.total_hits[q] <= wt[i])):
                raise SystemExit(f"{name}: GPU results differ from the reference (query {q})")

    def timed(run):
        for _ in range(a.warmup):
            run()
        ts = []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            run()   # every call copies its results to the host and synchronises
            ts.append(time.perf_counter() - t0)
        return ts

    def kernel_ms(prepared):
        for _ in range(a.warmup):
            prepared.run(); prepared.fetch()
        prepared.reset_timing()
        for _ in range(a.steps):
            prepared.run(); prepared.fetch()
        ms = prepared.stage_ms(0)
        items = prepared.stats()["work_items"]
        prepared.close()
        return ms, items

    workloads = [
        ("(a) match-in-bool + range, search_tree", tree, True),
        ("(b) flattened, msm 1, search_batch", flat, False),
        ("(c) multi_match BEST_FIELDS + range, tie 0", multi(0.0), True),
        ("(c) multi_match BEST_FIELDS + range, tie 0.3", multi(0.3), True),
    ]
    for name, queries, is_tree in workloads:
        run = (lambda q=queries: s.search_tree(q, col)) if is_tree else (lambda q=queries: s.search_batch(q, col))
        gate(name, run(), queries, is_tree)
        ts = timed(run)
        kms, items = kernel_ms(s.prepare_tree(queries, col) if is_tree else s.prepare(queries, col))
        med = float(np.median(ts))
        print(json.dumps({**base, "workload": name, "ms_median": round(1e3 * med, 3), "ms_min": round(1e3 * min(ts), 3),
                          "qps": round(nq / med, 1), "kernel_ms": round(kms, 3), "work_items": items, "steps": a.steps,
                          "oracle_gate": f"{len(sample)} queries bit-exact"}), flush=True)
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
