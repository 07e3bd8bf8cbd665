#!/usr/bin/env python
"""Keyword range clauses (NRTGPU_KEYWORD_RANGE) against numeric range clauses of the same shape, on bench.py's BM25 corpus:
10M docs, 1M-term vocabulary, 1024-query batches, top 100.

Keyword columns: SORTED of 20,000 terms with 10 % of docs without a value (`kw`), and SORTED_SET of 1-4 distinct
Zipf(1.3)-drawn terms of 1,000 per doc (about 2.3 per doc; `kw_set`). Each has a shadow numeric column of its codes
(single-valued with has = code != 0, and multi-valued), so a keyword clause and its twin NRTGPU_RANGE_I64 clause over the
same code range match the same docs. Workloads, each on `kw` and on `kw_set`, keyword leg alternated step by step with its
shadow-range twin:
  - "conj+range": a conjunction of 2-3 terms plus a keyword FILTER range covering about a third of the terms;
  - "conj+prefix": the same with a prefix (a third of the terms share it);
  - "kw-only sorted": the keyword range alone, sorted by a numeric column (search_sorted, top 100).
The scored workloads are prepared batches (TOP_SCORES, totalHitsThreshold 1000) timed from run to fetch with CUDA events;
the sorted one is a synchronous search_sorted call between two events. Before timing, each keyword leg's results are
checked bit-exact against its twin's. Prints one JSON line per leg (median, min, max over --steps), then the card's name,
power limit and SM clock read in the same run.
python tools/keyword_query_bench.py [--docs 10000000] [--vocab 1000000] [--nq 1024] [--k 100] [--steps 10] [--warmup 2]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def sorted_column(n, n_terms, rng):
    from nrtsearch_b200.index import KeywordColumn
    ords = rng.integers(0, n_terms, n).astype(np.int32)
    ords[rng.random(n) < 0.1] = -1
    return KeywordColumn(sorted(b"%c%05d" % (b"abc"[i % 3], i) for i in range(n_terms)), ords)


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
    return KeywordColumn(sorted(b"%c%04d" % (b"abc"[i % 3], i) for i in range(n_terms)), vals.astype(np.int32), off)


def stats(t):
    return {"ms_median": round(float(np.median(t)), 3), "ms_min": round(min(t), 3), "ms_max": round(max(t), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000); ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1024); ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch
    import __graft_entry__ as g
    g.build_if_needed()
    from nrtsearch_b200 import index as ix
    from nrtsearch_b200.search import (BooleanQuery, GpuContext, GpuIndex, GpuIndexSearcher, KeywordPrefixQuery, KeywordRangeQuery,
                                       Occur, RangeQuery, RelevanceCollector, SortFieldCollector, SortType, TermQuery)
    n, nq, k = a.docs, a.nq, a.k
    KW, KW_SET = 0, 1
    SHADOW, NUM = {KW: 0, KW_SET: 1}, 2
    rng = np.random.default_rng(0x4B51)
    sh = ix.synth_text_shard(n, a.vocab)
    kc = [sorted_column(n, 20_000, rng), sorted_set_column(n, 1_000, rng)]
    one = np.where(kc[0].ords < 0, 0, 2 * kc[0].ords.astype(np.int64) + 2)
    sh.columns = [one, 2 * kc[1].ords.astype(np.int64) + 2, rng.integers(0, 1_000_000, n).astype(np.int64)]
    sh.column_has = [(one != 0).astype(np.uint8), None, None]
    sh.column_offsets = [None, kc[1].offsets, None]
    sh.keyword_columns = kc
    terms = ix.synth_query_terms(nq, 3, a.vocab)
    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    base = {"docs": n, "vocab": a.vocab, "batch": nq, "top_k": k,
            "kw_set_terms_per_doc": round(float(np.diff(kc[1].offsets).mean()), 3)}

    def twin(kq):
        lo, hi = gix.keyword_range(kq)
        return RangeQuery(SHADOW[kq.column], lo, hi)

    def conj(i, kq):
        t = terms[i]
        b = BooleanQuery().add(TermQuery(int(t[0])), Occur.MUST).add(TermQuery(int(t[1])), Occur.MUST)
        if i % 2:
            b.add(TermQuery(int(t[2])), Occur.MUST)
        return b.add(kq, Occur.FILTER)

    def kw_range(col, i):   # about a third of the terms, starting at a drifting term
        lo = (i * 7) % 600 if col == KW_SET else (i * 131) % 12_000
        span = 333 if col == KW_SET else 6_667
        t = kc[col].terms
        return KeywordRangeQuery(col, t[lo].decode(), t[min(lo + span, len(t) - 1)].decode())

    def kw_prefix(col, i):
        return KeywordPrefixQuery(col, "abc"[i % 3])

    coll = RelevanceCollector(k, 1000)
    sort_coll = SortFieldCollector(k, SortType(NUM))
    for col, cname in ((KW, "kw (SORTED)"), (KW_SET, "kw_set (SORTED_SET)")):
        work = {"conj+range": [conj(i, kw_range(col, i)) for i in range(nq)],
                "conj+prefix": [conj(i, kw_prefix(col, i)) for i in range(nq)],
                "kw-only sorted": [kw_range(col, i) for i in range(nq)]}
        for wname, kqs in work.items():
            def twin_of(q):
                if isinstance(q, BooleanQuery):
                    b = BooleanQuery()
                    for c in q.clauses:
                        b.add(twin(c.query) if isinstance(c.query, (KeywordRangeQuery, KeywordPrefixQuery)) else c.query, c.occur)
                    return b
                return twin(q)
            legs = {"keyword": kqs, "shadow range": [twin_of(q) for q in kqs]}
            if wname == "kw-only sorted":
                res = {x: s.search_sorted(qs, sort_coll) for x, qs in legs.items()}
                r0, r1 = res["keyword"], res["shadow range"]
                ok = np.array_equal(r0.docs, r1.docs) and np.array_equal(r0.counts, r1.counts) and np.array_equal(r0.sort_values, r1.sort_values)
                run = {x: (lambda qs=qs: s.search_sorted(qs, sort_coll)) for x, qs in legs.items()}
            else:
                pbs = {x: s.prepare(qs, coll) for x, qs in legs.items()}
                res = {}
                for x, pb in pbs.items():
                    pb.run()
                    res[x] = pb.fetch()
                r0, r1 = res["keyword"], res["shadow range"]
                ok = all(np.array_equal(getattr(r0, f), getattr(r1, f)) for f in ("docs", "counts", "total_hits", "relation"))
                ok = ok and np.array_equal(r0.scores.view(np.uint32), r1.scores.view(np.uint32))
                run = {x: (lambda pb=pb: (pb.run(), pb.fetch())) for x, pb in pbs.items()}
            if not ok:
                raise SystemExit(f"{cname} {wname}: the keyword leg differs from its shadow-range twin")
            t = {x: [] for x in legs}
            for step in range(a.warmup + a.steps):
                for x in legs:   # alternated step by step: both legs share the card's state
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    run[x]()
                    e1.record()
                    e1.synchronize()
                    if step >= a.warmup:
                        t[x].append(e0.elapsed_time(e1))
            for x in legs:
                print(json.dumps({**base, "column": cname, "workload": wname, "leg": x, **stats(t[x]),
                                  "qps": round(nq / (float(np.median(t[x])) / 1e3), 1), "steps": a.steps}), flush=True)
            if wname != "kw-only sorted":
                for pb in pbs.values():
                    pb.close()
    print(json.dumps({"gpu": card()}), flush=True)
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
