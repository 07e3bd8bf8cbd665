#!/usr/bin/env python
"""Sorted search on several fields (nrtgpu_sort_order / nrtgpu_search_sorted_fields) on the bench corpus: 10M docs, 1M-term
vocabulary, 1024 three-term disjunctions (bench.py's default queries), top 100, plus synthetic int columns (0: the bench's
price column, 1: a rating in [0, 50), 2: a review count in [0, 10000), 3: a popularity in [0, 1000) missing on 30 % of the docs).
Prints one JSON line per measurement:
  - the order build time (nrtgpu_sort_order_create, synchronised) for a 2-field and a 4-field Sort;
  - the time of one 1024-query batch for relevance (totalHitsThreshold 1000, as bench.py), a single-field sort through
    nrtgpu_search_sorted, the two-column Sort [rating desc, review_count desc] and [score, popularity desc];
and the card name and power limit, read in the same run. Each workload is first checked on a sample of queries, bit-exact
on docs, every FieldDoc value (scores for relevance), counts and totals: against the oracle for relevance and the single
field, against tests/sort_fields_reference.py for Sorts of several fields. A failed check stops the run.
python tools/sort_fields_bench.py [--docs 10000000] [--vocab 1000000] [--nq 1024] [--k 100] [--steps 10] [--warmup 2] [--sample 8]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # sort_fields_reference: the multi-field checker


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the JSON still says what was measured on
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000); ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1024); ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=8, help="queries per sorted workload checked against the oracle")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build_if_needed()
    import oracle
    import sort_fields_reference as ref
    from nrtsearch_b200 import _native, index as ix
    from nrtsearch_b200.search import (BooleanQuery, GpuContext, GpuIndex, GpuIndexSearcher, Occur, RelevanceCollector,
                                       SortFieldCollector, SortType, TermQuery, compile_queries)
    n, nq, k = a.docs, a.nq, a.k
    sh = ix.synth_text_shard(n, a.vocab)
    rng = np.random.default_rng(23)
    sh.columns = [ix.synth_int_column(n), rng.integers(0, 50, n).astype(np.int64), rng.integers(0, 10_000, n).astype(np.int64),
                  rng.integers(0, 1_000, n).astype(np.int64)]
    sh.column_has = [None, None, None, (rng.random(n) < 0.7).astype(np.uint8)]
    terms = ix.synth_query_terms(nq, 3, a.vocab)
    queries = [BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD).add(TermQuery(int(t[1])), Occur.SHOULD)
               .add(TermQuery(int(t[2])), Occur.SHOULD) for t in terms]
    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    lib = _native.gpu_lib()
    gpu = card()
    base = {"docs": n, "vocab": a.vocab, "batch": nq, "top_k": k, "gpu": gpu}

    # order build (the adaptor builds one per (leaf, Sort) and reuses it)
    for name, spec in (("2 fields", [SortType(1, True), SortType(2, True)]),
                       ("4 fields", [SortType(1, True), SortType(2, True), SortType(3, False, True), SortType(0)])):
        cf = [f.c_field() for f in spec]
        arr = (_native.SortField * len(cf))(*cf)
        times = []
        for _ in range(a.warmup + a.steps):
            h = C.c_void_p()
            t0 = time.perf_counter()
            _native.check(lib.nrtgpu_sort_order_create(gix.handle, arr, len(cf), None, C.byref(h)))
            times.append(time.perf_counter() - t0)
            lib.nrtgpu_sort_order_close(h)
        t = times[a.warmup:]
        print(json.dumps({**base, "measure": "order build", "sort": name, "ms_median": round(1e3 * float(np.median(t)), 3),
                          "ms_min": round(1e3 * min(t), 3), "steps": a.steps}), flush=True)

    oix = oracle.OracleIndex(sh)
    sample = list(range(0, nq, max(1, nq // a.sample)))[:a.sample]
    carr, ncl, qarr, snq = compile_queries([queries[i] for i in sample])

    def gate(name, res, spec):
        sub = [queries[i] for i in sample]
        if isinstance(spec, SortType):
            wd, wv, wc, wt = oracle.search_sorted(oix, carr, ncl, qarr, snq, k, 2 if spec.field == "docid" else 1, spec.field,
                                                   spec.reverse, spec.missing_value(), n_threads=8)
            wv = wv[:, :, None]
            got_v = res.sort_values[sample][:, :, None]
        else:
            fields = [tuple(getattr(f.c_field(), x) for x in ("kind", "column", "reverse", "selector", "missing_value")) for f in spec]
            wd, wv, wc, wt = ref.search_sorted_fields(sh, carr, ncl, qarr, snq, k, fields, oix=oix)
            got_v = res.sort_values[sample]
        ok = np.array_equal(res.counts[sample], wc) and np.array_equal(res.total_hits[sample], wt)
        for i, q in enumerate(sample):
            c = wc[i]
            ok = ok and np.array_equal(res.docs[q, :c], wd[i, :c]) and np.array_equal(got_v[i, :c], wv[i, :c])
        if not ok:
            raise SystemExit(f"{name}: GPU results differ from the oracle on the sample ({len(sub)} queries)")

    def timed(run):
        for _ in range(a.warmup):
            run()
        t = []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            run()   # every call copies its results to the host and synchronises
            t.append(time.perf_counter() - t0)
        return t

    workloads = [
        ("relevance", lambda: s.search_batch(queries, RelevanceCollector(k, 1000)), None),
        ("single field (nrtgpu_search_sorted) [review_count desc]", lambda: s.search_sorted(queries, SortFieldCollector(k, SortType(2, True))),
         SortType(2, True)),
        ("two columns [rating desc, review_count desc]",
         lambda: s.search_sorted(queries, SortFieldCollector(k, [SortType(1, True), SortType(2, True)])), [SortType(1, True), SortType(2, True)]),
        ("[score, popularity desc]", lambda: s.search_sorted(queries, SortFieldCollector(k, [SortType("score"), SortType(3, True)])),
         [SortType("score"), SortType(3, True)]),
    ]
    for name, run, spec in workloads:
        res = run()
        if spec is not None:
            gate(name, res, spec)
        else:
            wd, ws, wc, _, _ = oracle.search_compiled(oix, carr, ncl, qarr, snq, k, n_threads=8)
            for i, q in enumerate(sample):
                c = wc[i]
                if not (res.counts[q] == c and np.array_equal(res.docs[q, :c], wd[i, :c])
                        and np.array_equal(res.scores[q, :c].view(np.uint32), ws[i, :c].view(np.uint32))):
                    raise SystemExit(f"{name}: GPU results differ from the oracle")
        t = timed(run)
        med = float(np.median(t))
        print(json.dumps({**base, "measure": "batch", "workload": name, "ms_median": round(1e3 * med, 3),
                          "ms_min": round(1e3 * min(t), 3), "qps": round(nq / med, 1), "steps": a.steps,
                          "oracle_gate": f"{len(sample)} queries bit-exact"}), flush=True)
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
