#!/usr/bin/env python
"""ConstantScoreQuery and MinScoreQuery nodes (nrtgpu_search_tree) on the 10M-doc bench shard (1M-term vocabulary, mean
length 56) with the bench's price column. Batches of 1024 queries, top 100, totalHitsThreshold 1000. Two pairs of
workloads, each wrapped tree against the same tree without the wrapper:
  (a) BooleanQuery(SHOULD match(t1, t2), SHOULD BoostQuery(ConstantScoreQuery(t3), 2)) against
      BooleanQuery(SHOULD match(t1, t2), SHOULD BoostQuery(t3, 2));
  (b) MinScoreQuery(match(t1, t2), t) against match(t1, t2), where t is the score at rank 50 of the query's unwrapped page.
      A bare match is a flat query, which the probe kernel runs; BooleanQuery(MUST match(t1, t2)) is the same query as a
      tree (a root over one node, as the wrapped query compiles), which the window engine runs, so it is timed too.
Every workload is first checked on a sample of queries, bit-exact on docs, scores, counts and totalHits, against
tests/score_nodes_reference.py (compiled arrays); a failed check stops the run. Prints one JSON line per workload with the batch time (host clock
around a call that ends with the results on the host), the search kernel time (CUDA events of a prepared batch, after
warm-up), and the card name and power limit read in the same run.
python tools/score_nodes_bench.py [--docs 10000000] [--nq 1024] [--k 100] [--steps 10] [--warmup 2] [--sample 8]"""
import argparse, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # score_nodes_reference: the checker of the trees
sys.path.insert(0, os.path.join(ROOT, "tools"))
from tree_bench import card   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1024); ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=8, help="queries per workload checked against the reference")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build_if_needed()
    import oracle
    import score_nodes_reference as ref
    from nrtsearch_b200 import index as ix
    from nrtsearch_b200.search import (BooleanQuery, BoostQuery, ConstantScoreQuery, GpuContext, GpuIndex, GpuIndexSearcher,
                                       MinScoreQuery, Occur, RelevanceCollector, TermQuery)
    n, nq, k = a.docs, a.nq, a.k
    sh = ix.synth_text_shard(n, a.vocab)
    sh.columns = [ix.synth_int_column(n)]
    sh.column_has = [None]
    t = ix.synth_query_terms(nq, 3, a.vocab)

    def match(x):
        return BooleanQuery().add(TermQuery(int(x[0])), Occur.SHOULD).add(TermQuery(int(x[1])), Occur.SHOULD)

    boosted = [BooleanQuery().add(match(x), Occur.SHOULD).add(BoostQuery(TermQuery(int(x[2])), 2.0), Occur.SHOULD) for x in t]
    constant = [BooleanQuery().add(match(x), Occur.SHOULD).add(BoostQuery(ConstantScoreQuery(TermQuery(int(x[2]))), 2.0), Occur.SHOULD)
                for x in t]
    plain = [match(x) for x in t]
    nested = [BooleanQuery().add(match(x), Occur.MUST) for x in t]

    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    gpu = card()
    base = {"docs": n, "batch": nq, "top_k": k, "threshold": 1000, "gpu": gpu}
    oix = oracle.OracleIndex(sh)
    sample = list(range(0, nq, max(1, nq // a.sample)))[:a.sample]
    col = RelevanceCollector(k, 1000)
    page = s.search_tree(plain, RelevanceCollector(50, 1000))
    thresholds = [float(page.scores[i, page.counts[i] - 1]) if page.counts[i] else 1.0 for i in range(nq)]
    min_score = [MinScoreQuery(q, th) for q, th in zip(plain, thresholds)]

    def gate(name, res, queries):
        sub = [queries[i] for i in sample]
        wd, ws, wc, wt, _ = ref.search(sh, sub, k, oix=oix)
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
        ("(a) match + SHOULD BoostQuery(term, 2)", boosted),
        ("(a) match + SHOULD BoostQuery(ConstantScoreQuery(term), 2)", constant),
        ("(b) match", plain),
        ("(b) BooleanQuery(MUST match)", nested),
        ("(b) MinScoreQuery(match, rank-50 score)", min_score),
    ]
    for name, queries in workloads:
        run = lambda q=queries: s.search_tree(q, col)   # noqa: E731
        gate(name, run(), queries)
        ts = timed(run)
        kms, items = kernel_ms(s.prepare_tree(queries, col))
        med = float(np.median(ts))
        print(json.dumps({**base, "workload": name, "ms_median": round(1e3 * med, 3), "ms_min": round(1e3 * min(ts), 3),
                          "qps": round(nq / med, 1), "kernel_ms": round(kms, 3), "work_items": items,
                          "steps": a.steps, "oracle_gate": f"{len(sample)} queries bit-exact"}), flush=True)
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
