#!/usr/bin/env python
"""Typeahead (match_phrase_prefix, MultiPhraseQuery leaves: nrtgpu_search_tree_phrases with NRTGPU_MULTI_PHRASE clauses) on
tools/phrase_bench.py's 10M-doc two-field shard with positions. A prefix is a run of 50 consecutive field-1 term ids (the
terms a sorted dictionary seek would enumerate), drawn from 64 prefixes per workload, so that the 1024 queries of a batch
share their unions as typeahead traffic does:
  (a) one token: the prefix alone (the disjunction of its 50 expansions);
  (b) two tokens: a field-1 token of a random doc followed by the prefix holding that doc's next token; the first token
      is one of at most 2,000 docs (a rarer word leads: the sample's reference check walks its docs in Python).
Every workload is first checked on a sample of queries, bit-exact on docs, scores, counts and totalHits, against
tests/multi_phrase_reference.py; a failed check stops the run. Prints one JSON line per workload: the host-clock batch time
(a call that ends with the results on the host) and the part of it spent compiling the query objects in Python
(compile_tree), the union build and the window engine split from CUDA kernel times (torch.profiler over separate calls:
the union_* and cub kernels against bool_window_union_kernel), and the card's name, power limit and SM clock read in the
same run.
python tools/phrase_prefix_bench.py [--docs 10000000] [--nq 1024] [--k 10] [--steps 10] [--warmup 2] [--sample 6]"""
import argparse, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from phrase_bench import field0_positions, field1_tokens   # noqa: E402
from tree_bench import card   # noqa: E402

FAMILY = 50


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000); ap.add_argument("--vocab1", type=int, default=100_000)
    ap.add_argument("--nq", type=int, default=1024); ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=6, help="distinct queries per workload checked against the reference")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build_if_needed()
    import torch
    import oracle
    import multi_phrase_reference as ref
    import phrase_reference as pr
    from nrtsearch_b200 import index as ix
    from nrtsearch_b200.search import (GpuContext, GpuIndex, GpuIndexSearcher, MatchPhrasePrefixQuery, RelevanceCollector,
                                       compile_tree)
    n, nq, k = a.docs, a.nq, a.k
    rng = np.random.default_rng(23)
    log = lambda m: print(f"[phrase_prefix_bench] {m}", file=sys.stderr, flush=True)   # noqa: E731  (progress of the slow set-up)
    log("building the shard")
    f0 = ix.synth_text_shard(n, a.vocab)
    lut = np.array([oracle.byte4_to_int(b) for b in range(256)], np.int64)
    pos0 = field0_positions(f0, lut[f0.fields[0].norms])
    doc1, tok1, p1, start1 = field1_tokens(n, a.vocab1, rng)
    f1 = pr.shard_from_token_arrays(n, np.zeros(a.vocab1, np.int32), 1, doc1, tok1, p1)
    sh = ix.HostShard(n_docs=n, doc_base=0, term_off=np.concatenate([f0.term_off, f0.term_off[-1] + f1.term_off[1:]]),
                      post_docs=np.concatenate([f0.post_docs, f1.post_docs]), post_freqs=np.concatenate([f0.post_freqs, f1.post_freqs]),
                      fields=[f0.fields[0], f1.fields[0]],
                      term_field=np.concatenate([np.zeros(a.vocab, np.int32), np.ones(a.vocab1, np.int32)]),
                      post_positions=np.concatenate([pos0, f1.post_positions]))
    sh.term_df = np.diff(sh.term_off).astype(np.int64)
    del f0, f1, pos0

    def family(t):   # the 50 ids of the prefix that holds field-1 term t
        lo = min((t // FAMILY) * FAMILY, a.vocab1 - FAMILY)
        return [a.vocab + lo + i for i in range(FAMILY)]

    one, two = [], []
    while len(two) < 64:
        d = int(rng.integers(0, n))
        if start1[d + 1] - start1[d] < 2:
            continue
        s = int(rng.integers(0, start1[d + 1] - start1[d] - 1))
        t0, t1 = int(tok1[start1[d] + s]), int(tok1[start1[d] + s + 1])
        if a.vocab + t0 in family(t1) or sh.term_df[a.vocab + t0] > 2000:
            continue
        one.append(MatchPhrasePrefixQuery([], family(t1)))
        two.append(MatchPhrasePrefixQuery([[a.vocab + t0]], family(t1)))
    workloads = [("(a) one-token prefix, 50 expansions", one), ("(b) two-token prefix, 50 expansions", two)]
    log("uploading the image")
    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    oix = oracle.OracleIndex(sh)
    col = RelevanceCollector(k, 2**31 - 1)
    base = {"docs": n, "batch": nq, "top_k": k, "distinct_prefixes": 64, "expansions": FAMILY, "gpu": card()}
    for name, shapes in workloads:
        pick = rng.integers(0, len(shapes), nq)
        queries = [shapes[int(i)] for i in pick]
        res = s.search_tree(queries, col)
        sample = sorted({int(i) for i in pick[:a.sample]})
        log(f"{name}: checking {len(sample)} queries against the reference")
        wd, ws, wc, wt, _ = ref.search(sh, [shapes[i] for i in sample], k, oix=oix)
        for j, i in enumerate(sample):
            q = int(np.nonzero(pick == i)[0][0])
            c = wc[j]
            if not (res.counts[q] == c and np.array_equal(res.docs[q, :c], wd[j, :c]) and res.total_hits[q] == wt[j]
                    and np.array_equal(res.scores[q, :c].view(np.uint32), ws[j, :c].view(np.uint32))):
                raise SystemExit(f"{name}: GPU results differ from the reference (query {q})")
        for _ in range(a.warmup):
            s.search_tree(queries, col)
        ts = []
        for _ in range(a.steps):
            t = time.perf_counter()
            s.search_tree(queries, col)   # every call builds its unions, searches and copies its results to the host
            ts.append(time.perf_counter() - t)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
            for _ in range(a.steps):
                s.search_tree(queries, col)
        build = engine = other = 0.0
        for e in prof.key_averages():
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if "bool_window" in e.key:   # (bool_window_union_kernel: before the union_ test)
                engine += us
            elif "union_" in e.key or "cub::" in e.key or "DeviceRadixSort" in e.key or "DeviceScan" in e.key:
                build += us
            else:
                other += us
        cts = []
        for _ in range(a.steps):
            t = time.perf_counter()
            compile_tree(queries, phrase_table=True)
            cts.append(time.perf_counter() - t)
        med = float(np.median(ts))
        import subprocess
        clk = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True).stdout.strip()
        print(json.dumps({**base, "sm_clock_after": clk, "workload": name, "ms_median": round(1e3 * med, 3), "ms_min": round(1e3 * min(ts), 3),
                          "qps": round(nq / med, 1),
                          "python_compile_ms": round(1e3 * float(np.median(cts)), 3), "union_build_ms": round(build / 1e3 / a.steps, 3),
                          "window_engine_ms": round(engine / 1e3 / a.steps, 3), "other_kernels_ms": round(other / 1e3 / a.steps, 3),
                          "matching_queries": int((res.total_hits > 0).sum()), "steps": a.steps,
                          "oracle_gate": f"{len(sample)} distinct queries bit-exact"}), flush=True)
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
