#!/usr/bin/env python
"""Block joins (NestedQuery: nrtgpu_search_tree with NRTGPU_NODE_NESTED nodes) on a synthetic nested index: about 2.5M
parents, each after a Poisson(3) number of child docs (about 10M docs), the children on two paths (70 % / 30 %), every doc
with a Zipf-like text field. Every query carries the root filter {FILTER _nested_path:_root, MUST q} the reference puts on
the top-level query of an index with nested fields. Three 1024-query workloads of selective child terms (ranks 100 ..
5,000, so a batch's child matches stay under the 2^26 join cap):
  (a) a nested child term, at SUM and at MAX;
  (b) a parent term MUST plus a nested child term SHOULD, at AVG;
  (c) a nested child bool: a term MUST, a term SHOULD and a range FILTER, at SUM.
Every workload is first checked on a sample of queries, bit-exact on docs, scores, counts and totalHits, against
tests/nested_reference.py; a failed check stops the run. Prints one JSON line per workload: the host-clock batch time (a
call that ends with the results on the host), the CUDA kernel times of the child pass (bool_window_emit_kernel), the
fold (join_* and the CUB sort and scan) and the parent pass (bool_window_union_kernel), from torch.profiler over separate
calls, and the card's name, power limit and SM clock read in the same run.
python tools/nested_bench.py [--parents 2500000] [--nq 1024] [--k 10] [--steps 10] [--warmup 2] [--sample 4]"""
import argparse, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from tree_bench import card   # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parents", type=int, default=2_500_000)
    ap.add_argument("--vocab", type=int, default=50_000)
    ap.add_argument("--nq", type=int, default=1024); ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=4, help="queries per workload checked against the reference")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build_if_needed()
    import nested_reference as nr
    from nrtsearch_b200.search import (BooleanQuery, GpuContext, GpuIndex, GpuIndexSearcher, NestedQuery, Occur, RangeQuery,
                                       RelevanceCollector, TermQuery)
    log = lambda m: print(f"[nested_bench] {m}", file=sys.stderr, flush=True)   # noqa: E731  (progress of the slow set-up)
    log("building the shard")
    sh, paths = nr.build_nested_shard(a.parents, 41, vocab=a.vocab, trailing=0, parents_on_path=0)
    root = sh.parent_term
    rng = np.random.default_rng(5)
    df = np.diff(sh.term_off)
    by_df = np.argsort(-df[:a.vocab], kind="stable")
    child_terms = by_df[100:5000]

    def t():
        return TermQuery(int(rng.choice(child_terms)))

    def filtered(q):
        return BooleanQuery().add(TermQuery(root), Occur.FILTER).add(q, Occur.MUST)

    def w_a(mode):
        return [filtered(NestedQuery(t(), paths[0], mode)) for _ in range(a.nq)]

    def w_b():
        return [filtered(BooleanQuery().add(TermQuery(int(rng.choice(by_df[20:2000]))), Occur.MUST)
                         .add(NestedQuery(t(), paths[0], "avg"), Occur.SHOULD)) for _ in range(a.nq)]

    def w_c():
        out = []
        for _ in range(a.nq):
            lo = int(rng.integers(0, 800_000))
            child = BooleanQuery().add(t(), Occur.MUST).add(t(), Occur.SHOULD).add(RangeQuery(0, lo, lo + 200_000), Occur.FILTER)
            out.append(filtered(NestedQuery(child, paths[0], "sum")))
        return out

    workloads = [("(a) nested child term, SUM", w_a("sum")), ("(a) nested child term, MAX", w_a("max")),
                 ("(b) parent term MUST + nested child term SHOULD, AVG", w_b()),
                 ("(c) nested child bool of two terms + range, SUM", w_c())]
    log("uploading the image")
    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    ref = nr.NestedReference(sh)
    col = RelevanceCollector(a.k, 2**31 - 1)
    base = {"docs": sh.n_docs, "parents": a.parents, "batch": a.nq, "top_k": a.k, "gpu": card()}
    for name, queries in workloads:
        res = s.search_tree(queries, col)
        log(f"{name}: checking {a.sample} queries against the reference")
        wd, ws, wc, wt = ref.search(queries[:a.sample], a.k)
        for q in range(a.sample):
            c = wc[q]
            if not (res.counts[q] == c and np.array_equal(res.docs[q, :c], wd[q, :c]) and res.total_hits[q] == wt[q]
                    and np.array_equal(res.scores[q, :c].view(np.uint32), ws[q, :c].view(np.uint32))):
                raise SystemExit(f"{name}: GPU results differ from the reference (query {q})")
        for _ in range(a.warmup):
            s.search_tree(queries, col)
        ts = []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            s.search_tree(queries, col)   # every call builds its joins, searches and copies its results to the host
            ts.append(time.perf_counter() - t0)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            for _ in range(a.steps):
                s.search_tree(queries, col)
        child = fold = parent = other = 0.0
        for e in prof.key_averages():
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if "bool_window_emit" in e.key:
                child += us
            elif "bool_window" in e.key:
                parent += us
            elif "join_" in e.key or "cub::" in e.key or "DeviceRadixSort" in e.key or "DeviceScan" in e.key:
                fold += us
            else:
                other += us
        med = float(np.median(ts))
        clk = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True).stdout.strip()
        print(json.dumps({**base, "sm_clock_after": clk, "workload": name, "ms_median": round(1e3 * med, 3),
                          "ms_min": round(1e3 * min(ts), 3), "qps": round(a.nq / med, 1),
                          "child_pass_ms": round(child / 1e3 / a.steps, 3), "fold_ms": round(fold / 1e3 / a.steps, 3),
                          "parent_pass_ms": round(parent / 1e3 / a.steps, 3), "other_kernels_ms": round(other / 1e3 / a.steps, 3),
                          "matching_queries": int((res.total_hits > 0).sum()), "steps": a.steps,
                          "oracle_gate": f"{a.sample} queries bit-exact"}), flush=True)
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
