#!/usr/bin/env python
"""Keyword sort fields (NRTGPU_SORT_KEYWORD) against numeric sort fields of the same shape, on bench.py's BM25 corpus: 10M docs,
1M-term vocabulary, 1024 three-term disjunctions per batch, top 100.

Columns: an int column of 20,000 values (`num`, the numeric twin of the SORTED column), an int rating in [0, 50) (`rating`);
a SORTED keyword column of 20,000 terms with 10 % of docs without a value (`kw`), and a SORTED_SET column of 1-4 distinct
Zipf(1.3)-drawn terms of 1,000 per doc (about 2.3 per doc, the shape of tools/keyword_aggs_bench.py; `kw_set`).
Prints one JSON line per measurement:
  - order build (nrtgpu_sort_order_create, synchronised) of [kw], [kw_set min] and [num], alternated step by step;
  - one 1024-query batch of search_sorted by [kw], [kw, rating], [score, kw] alternated step by step with [num],
    [num, rating], [score, num], on one image and over three doc-range leaves (GpuLeafSearcher) of the same docs. Each
    call is synchronous and ends with its results on the host (keyword values as str), host work included;
then the card's name, power limit and SM clock, read in the same run. Before timing, every keyword workload is checked
on a sample of queries against tests/keyword_sort_reference.py, bit-exact on docs, FieldDoc values, counts and totals, and
the leaves' pages against the image's. A failed check stops the run. Each line gives the median, min and max over --steps.
python tools/keyword_sort_bench.py [--docs 10000000] [--vocab 1000000] [--nq 1024] [--k 100] [--steps 10] [--warmup 2] [--sample 4]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # keyword_sort_reference: the checker


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError) as e:   # the JSON still says what was measured on
        return f"unknown ({e})"


def sorted_column(n, n_terms, rng):
    from nrtsearch_b200.index import KeywordColumn
    ords = rng.integers(0, n_terms, n).astype(np.int32)
    ords[rng.random(n) < 0.1] = -1
    return KeywordColumn([b"s%05d" % i for i in range(n_terms)], ords)


def sorted_set_column(n, n_terms, rng):
    """1-4 distinct Zipf-drawn ordinals per doc, ascending"""
    from nrtsearch_b200.index import KeywordColumn
    per = rng.integers(1, 5, n)
    owner = np.repeat(np.arange(n, dtype=np.int64), per)
    vals = (rng.zipf(1.3, size=len(owner)) - 1) % n_terms
    order = np.lexsort((vals, owner))
    owner, vals = owner[order], vals[order]
    keep = np.ones(len(vals), bool)
    keep[1:] = (owner[1:] != owner[:-1]) | (vals[1:] != vals[:-1])
    owner, vals = owner[keep], vals[keep]
    off = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(owner, minlength=n), out=off[1:])
    return KeywordColumn([b"k%05d" % i for i in range(n_terms)], vals.astype(np.int32), off)


def stats(t):
    return {"ms_median": round(1e3 * float(np.median(t)), 3), "ms_min": round(1e3 * min(t), 3), "ms_max": round(1e3 * max(t), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000); ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1024); ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sample", type=int, default=4, help="queries per keyword workload checked against the reference")
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build_if_needed()
    import keyword_sort_reference as ref
    from nrtsearch_b200 import _native, index as ix
    from nrtsearch_b200.search import (BooleanQuery, GpuContext, GpuIndex, GpuIndexSearcher, GpuLeafSearcher, Occur,
                                       SortFieldCollector, SortType, TermQuery, compile_queries)
    n, nq, k = a.docs, a.nq, a.k
    NUM, RATING, KW, KW_SET = 0, 1, 0, 1
    rng = np.random.default_rng(0x4B53)
    sh = ix.synth_text_shard(n, a.vocab)
    sh.columns = [rng.integers(0, 20_000, n).astype(np.int64), rng.integers(0, 50, n).astype(np.int64)]
    sh.column_has = [None, None]
    sh.keyword_columns = [sorted_column(n, 20_000, rng), sorted_set_column(n, 1_000, rng)]
    terms = ix.synth_query_terms(nq, 3, a.vocab)
    queries = [BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD).add(TermQuery(int(t[1])), Occur.SHOULD)
               .add(TermQuery(int(t[2])), Occur.SHOULD) for t in terms]
    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    cuts = [0, n // 3, (2 * n) // 3, n]
    leaves = [GpuIndex(ctx, sh.doc_range(lo, hi)) for lo, hi in zip(cuts, cuts[1:])]
    ls = GpuLeafSearcher(ctx, leaves)
    s = GpuIndexSearcher(gix)
    lib = _native.gpu_lib()
    vpd = float(np.diff(sh.keyword_columns[KW_SET].offsets).mean())
    base = {"docs": n, "vocab": a.vocab, "batch": nq, "top_k": k, "kw_set_terms_per_doc": round(vpd, 3)}

    # order build, the three Sorts alternated step by step (the adaptor builds one per (leaf, Sort) and reuses it)
    builds = {"[kw] (SORTED)": [SortType(KW, field_type="keyword")],
              "[kw_set min] (SORTED_SET)": [SortType(KW_SET, field_type="keyword")],
              "[num]": [SortType(NUM, field_type="int")]}
    times = {name: [] for name in builds}
    for step in range(a.warmup + a.steps):
        for name, spec in builds.items():
            cf = [f.c_field() for f in spec]
            arr = (_native.SortField * len(cf))(*cf)
            h = C.c_void_p()
            t0 = time.perf_counter()
            _native.check(lib.nrtgpu_sort_order_create(gix.handle, arr, len(cf), None, C.byref(h)))
            dt = time.perf_counter() - t0
            lib.nrtgpu_sort_order_close(h)
            if step >= a.warmup:
                times[name].append(dt)
    for name, t in times.items():
        print(json.dumps({**base, "measure": "order build", "sort": name, **stats(t), "steps": a.steps}), flush=True)

    kw, num = SortType(KW, field_type="keyword"), SortType(NUM, field_type="int")
    rating, score = SortType(RATING, True, field_type="int"), SortType("score")
    pairs = [("[kw]", [kw], "[num]", [num]), ("[kw, rating desc]", [kw, rating], "[num, rating desc]", [num, rating]),
             ("[score, kw]", [score, kw], "[score, num]", [score, num])]

    # the keyword workloads checked before they are timed: the image against the reference, the leaves against the image
    sample = list(range(0, nq, max(1, nq // a.sample)))[:a.sample]
    carr, ncl, qarr, snq = compile_queries([queries[i] for i in sample])
    for name, spec, _, _ in pairs:
        fields = [tuple(getattr(f.c_field(), x) for x in ("kind", "column", "reverse", "selector", "missing_value")) for f in spec]
        wd, wv, wc, wt = ref.search(sh, carr, ncl, qarr, snq, k, fields)
        res = s.search_sorted(queries, SortFieldCollector(k, spec))
        ok = np.array_equal(res.counts[sample], wc) and np.array_equal(res.total_hits[sample], wt)
        for i, q in enumerate(sample):
            c = wc[i]
            got = [tuple(x.encode() if isinstance(x, str) else x for x in row) for row in res.sort_values[q, :c]]
            ok = ok and np.array_equal(res.docs[q, :c], wd[i, :c]) and got == [tuple(row) for row in wv[i, :c]]
        lv = ls.search_sorted(queries, SortFieldCollector(k, spec))
        ok = ok and np.array_equal(lv.docs, res.docs) and np.array_equal(lv.counts, res.counts)
        ok = ok and list(lv.sort_values.reshape(-1)) == list(res.sort_values.reshape(-1))
        if not ok:
            raise SystemExit(f"{name}: GPU results differ from the reference on the sample ({len(sample)} queries)")

    for where, searcher in (("one image", s), ("three leaves", ls)):
        for kname, kspec, nname, nspec in pairs:
            legs = [(kname, kspec), (nname, nspec)]
            t = {x: [] for x, _ in legs}
            for step in range(a.warmup + a.steps):
                for x, spec in legs:   # alternated step by step: both legs share the card's state
                    t0 = time.perf_counter()
                    searcher.search_sorted(queries, SortFieldCollector(k, spec))
                    dt = time.perf_counter() - t0
                    if step >= a.warmup:
                        t[x].append(dt)
            for x, _ in legs:
                med = float(np.median(t[x]))
                print(json.dumps({**base, "measure": "batch", "on": where, "sort": x, **stats(t[x]), "qps": round(nq / med, 1),
                                  "steps": a.steps}), flush=True)
    print(json.dumps({"gpu": card()}), flush=True)
    ls.close()
    for g_ in leaves:
        g_.close()
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
