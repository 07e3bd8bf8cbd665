#!/usr/bin/env python
"""One image against a searcher over 8 leaves (nrtgpu_searcher_*) on the bench corpus: 10M docs, 1M-term vocabulary, 1024
queries, top 100, cut into 8 doc-range leaves of unequal size. Three batches:
  - sorted: the bench's three-term disjunctions under the Sort [rating desc, review_count desc] (nrtgpu_search_sorted_fields
    on one image, nrtgpu_searcher_search_sorted_fields over the leaves);
  - tree: a DisjunctionMaxQuery of two terms (tie 0.1) in a BooleanQuery with a third SHOULD term (nrtgpu_search_tree on one
    image, nrtgpu_searcher_search_tree_phrases over the leaves);
  - aggs: the three-term disjunctions with a terms aggregation on review_count (10,000 values, size 10) holding a nested max
    of rating and nested top 5 hits (nrtgpu_search_bool_aggs_nested on one image, nrtgpu_searcher_search_bool_aggs_nested over
    the leaves). The first call of a new searcher, which builds its reader-wide dictionary of the column, is reported apart
    from the steady state.
Each call is timed by the host clock around a device synchronise (every call returns host results). The sorted merge kernel
(nrtgpu_merge_sorted_packed over the 8 leaves' records of the same batch) is timed alone with CUDA events, and its share of
the 8-leaf call is reported. Before timing, the 8-leaf results are checked against the one-image results (docs, values or
score bits, counts, totals, and every aggregation output): a mismatch stops the run. Prints one JSON line per measurement with
the card and power limit.
python tools/searcher_leaves_bench.py [--docs 10000000] [--vocab 1000000] [--nq 1024] [--k 100] [--leaves 8] [--steps 10] [--warmup 2]
                                      [--workloads sorted,tree,aggs,merge]"""
import argparse, ctypes as C, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:   # the JSON still says what was measured on
        return f"unknown ({e})"


def timed(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), float(min(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000); ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1024); ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--leaves", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10); ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workloads", default="sorted,tree,aggs,merge")
    a = ap.parse_args()
    run = set(a.workloads.split(","))
    import torch
    import __graft_entry__ as g
    g.build_if_needed()
    from nrtsearch_b200 import _native, index as ix
    from nrtsearch_b200.search import (BooleanQuery, DisjunctionMaxQuery, GpuContext, GpuIndex, GpuIndexSearcher, GpuLeafSearcher,
                                       MaxCollector, Occur, RelevanceCollector, SortFieldCollector, SortType, TermQuery, TermsCollector,
                                       TopHitsCollector, compile_queries)
    from nrtsearch_b200.shards import SortedPackedGather
    n, nq, k, L = a.docs, a.nq, a.k, a.leaves
    sh = ix.synth_text_shard(n, a.vocab)
    rng = np.random.default_rng(23)
    sh.columns = [rng.integers(0, 50, n).astype(np.int64), rng.integers(0, 10_000, n).astype(np.int64)]
    sh.column_has = [None, None]
    w = rng.uniform(0.5, 1.5, L)                                  # unequal leaves, as segments of a live shard are
    cuts = np.concatenate([[0], np.round(np.cumsum(w) / w.sum() * n).astype(np.int64)])
    cuts[-1] = n
    terms = ix.synth_query_terms(nq, 3, a.vocab)
    flat = [BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD).add(TermQuery(int(t[1])), Occur.SHOULD)
            .add(TermQuery(int(t[2])), Occur.SHOULD) for t in terms]
    trees = [BooleanQuery().add(DisjunctionMaxQuery([TermQuery(int(t[0])), TermQuery(int(t[1]))], 0.1), Occur.SHOULD)
             .add(TermQuery(int(t[2])), Occur.SHOULD) for t in terms]
    ctx = GpuContext(0)
    whole = GpuIndex(ctx, sh)
    leaves = [GpuIndex(ctx, sh.doc_range(int(lo), int(hi))) for lo, hi in zip(cuts[:-1], cuts[1:])]
    one, many = GpuIndexSearcher(whole), GpuLeafSearcher(ctx, leaves)
    sort = [SortType(0, True, field_type="int"), SortType(1, True, field_type="int")]
    base = {"docs": n, "vocab": a.vocab, "batch": nq, "top_k": k, "leaves": L, "gpu": card()}

    # the leaves must answer what one image answers
    if "sorted" in run or "merge" in run:
        r1, rL = one.search_sorted(flat, SortFieldCollector(k, sort)), many.search_sorted(flat, SortFieldCollector(k, sort))
        for x, y in ((r1.docs, rL.docs), (r1.sort_values, rL.sort_values), (r1.counts, rL.counts), (r1.total_hits, rL.total_hits)):
            if not np.array_equal(x, y):
                sys.exit("sorted: the leaves differ from one image")
    if "tree" in run:
        t1, tL = one.search_tree(trees, RelevanceCollector(k)), many.search_tree(trees, RelevanceCollector(k))
        for q in range(nq):
            c = t1.counts[q]
            if c != tL.counts[q] or not np.array_equal(t1.docs[q, :c], tL.docs[q, :c]) or \
                    not np.array_equal(t1.scores[q, :c].view(np.uint32), tL.scores[q, :c].view(np.uint32)):
                sys.exit(f"tree: the leaves differ from one image at query {q}")
    adds = [TermsCollector(1, 10, True, "int", (("max", MaxCollector(0, "int")), ("hits", TopHitsCollector(5))))]
    if "aggs" in run:   # the first call of a new searcher builds its dictionary of the column
        fresh = GpuLeafSearcher(ctx, leaves)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gL = fresh.search_with_collectors(flat, RelevanceCollector(k), adds)
        first = (time.perf_counter() - t0) * 1e3
        fresh.close()
        g1 = one.search_with_collectors(flat, RelevanceCollector(k), adds)
        o1, oL = g1[1][0], gL[1][0]
        same = np.array_equal(g1[0].counts, gL[0].counts) and np.array_equal(g1[0].total_hits, gL[0].total_hits)
        for q, c in enumerate(g1[0].counts.tolist()):   # (a single-image page leaves the slots past the count unset)
            same &= np.array_equal(g1[0].docs[q, :c], gL[0].docs[q, :c])
            same &= np.array_equal(g1[0].scores[q, :c].view(np.uint32), gL[0].scores[q, :c].view(np.uint32))
        same &= all(np.array_equal(o1[f], oL[f]) for f in ("keys", "counts", "n", "total_buckets", "other_counts"))
        same &= np.array_equal(o1["nested"]["max"].view(np.uint64), oL["nested"]["max"].view(np.uint64))
        h1, hL = o1["nested"]["hits"], oL["nested"]["hits"]
        same &= all(np.array_equal(h1[f], hL[f]) for f in ("docs", "counts", "total_hits"))
        same &= np.array_equal(h1["scores"].view(np.uint32), hL["scores"].view(np.uint32))
        if not same:
            sys.exit("aggs: the leaves differ from one image")

    work = [("sorted", lambda: one.search_sorted(flat, SortFieldCollector(k, sort)), lambda: many.search_sorted(flat, SortFieldCollector(k, sort))),
            ("tree", lambda: one.search_tree(trees, RelevanceCollector(k)), lambda: many.search_tree(trees, RelevanceCollector(k))),
            ("aggs", lambda: one.search_with_collectors(flat, RelevanceCollector(k), adds),
             lambda: many.search_with_collectors(flat, RelevanceCollector(k), adds))]
    for name, f1, fL in work:
        if name not in run:
            continue
        m1, b1 = timed(f1, a.steps, a.warmup)
        mL, bL = timed(fL, a.steps, a.warmup)
        extra = {"leaves_first_call_ms": round(first, 3)} if name == "aggs" else {}
        print(json.dumps(dict(base, workload=name, one_image_ms=round(m1, 3), one_image_best_ms=round(b1, 3),
                              leaves_ms=round(mL, 3), leaves_best_ms=round(bL, 3), ratio=round(mL / m1, 3), **extra)), flush=True)

    # the sorted merge alone: the 8 leaves' records of the same batch, merged on the device, CUDA events around the launch
    if "merge" in run:
        lib = _native.gpu_lib()
        dev = torch.device("cuda", 0)
        pg = SortedPackedGather(nq, k, sort, L, dev)
        carr, ncl, qarr, _ = compile_queries(flat)
        for leaf, part in zip(leaves, pg.all.view(L, pg.words)):
            _native.check(lib.nrtgpu_search_sorted_fields_packed(leaf.handle, leaf.sort_order(sort), carr, ncl, qarr, nq, k, 0, None, None,
                                                                  None, part.data_ptr()))
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ms = []
        for i in range(a.warmup + a.steps):
            ev[0].record()
            pg.merge_on_device(ctx, torch.cuda.current_stream().cuda_stream)
            ev[1].record()
            torch.cuda.synchronize()
            if i >= a.warmup:
                ms.append(ev[0].elapsed_time(ev[1]))
        d, v, c, _, tot = pg.unpack()
        if not (np.array_equal(d, rL.docs) and np.array_equal(v, rL.sort_values) and np.array_equal(c, rL.counts)):
            sys.exit("sorted merge: the merged record differs from the searcher's page")
        mL, _ = timed(lambda: many.search_sorted(flat, SortFieldCollector(k, sort)), a.steps, a.warmup)
        merge = float(np.median(ms))
        print(json.dumps(dict(base, workload="sorted merge kernel", merge_ms=round(merge, 4), share_of_leaves_call=round(merge / mL, 4))),
              flush=True)
    many.close()
    for x in leaves + [whole]:
        x.close()
    ctx.close()


if __name__ == "__main__":
    main()
