#!/usr/bin/env python
"""Collectors on the window engine (nrtgpu_search_tree_aggs): tools/tree_bench.py's 10M-doc two-field shard and its price
column, plus a category column (the price folded to 1000 values) to bucket on. Batches of 1024 queries, top 100, exact
totalHits, workloads (a) match-in-bool + range and (c) multi_match BEST_FIELDS + range at tie 0.3 of tree_bench. Each
workload runs three legs, on one image and on 8 leaves (GpuLeafSearcher):
  plain:  search_tree at totalHitsThreshold INT32_MAX (no collectors; the same page as the other legs);
  terms:  search_tree_with_collectors with a size-10 terms aggregation on the category column and its top 3 hits;
  filter: the same plus FilterCollector(price range) with the same terms aggregation and top 3 nested in it.
Before timing, a sample of queries of every collector leg is checked against the references (rescore_tree_reference's
match sets and scores, nested_aggs_reference, filter_aggs_reference): bucket keys, counts, top-hit docs and score bits
exact; a failed check stops the run. Each timed call is a host clock around a call that ends with its results on the host
(compile, upload, both passes and the selection included). Prints one JSON line per (workload, target) with the median
and min of each leg, and the card name and power limit read in the same run.
python tools/tree_aggs_bench.py [--docs 10000000] [--nq 1024] [--k 100] [--steps 5] [--warmup 1] [--sample 4] [--leaves 8]"""
import argparse, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # the references
sys.path.insert(0, os.path.join(ROOT, "tools"))
from tree_bench import card, two_field_shard  # noqa: E402

INT_MAX = 2**31 - 1
CAT = 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000); ap.add_argument("--vocab1", type=int, default=100_000)
    ap.add_argument("--nq", type=int, default=1024); ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=5); ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=4, help="queries per collector leg checked against the references")
    ap.add_argument("--leaves", type=int, default=8)
    a = ap.parse_args()
    import __graft_entry__ as g
    g.build_if_needed()
    import filter_aggs_reference as far
    import nested_aggs_reference as nr
    import oracle
    import rescore_tree_reference as rtr
    from nrtsearch_b200 import index as ix
    from nrtsearch_b200.search import (BooleanQuery, DisjunctionMaxQuery, FilterCollector, GpuContext, GpuIndex, GpuIndexSearcher,
                                       GpuLeafSearcher, Occur, RangeQuery, RelevanceCollector, TermQuery, TermsCollector,
                                       TopHitsCollector, compile_queries)
    n, nq, k = a.docs, a.nq, a.k
    sh = two_field_shard(n, a.vocab, a.vocab1)
    sh.columns = [sh.columns[0], np.asarray(sh.columns[0], np.int64) % 1000]
    sh.column_has = [None, None]
    t = ix.synth_query_terms(nq, 2, a.vocab)
    u = ix.synth_query_terms(nq, 2, a.vocab1, seed=ix.SEED_QUERIES + 1) + a.vocab
    price = RangeQuery(0, 100_000, 600_000)
    fprice = RangeQuery(0, 200_000, 400_000)

    def match(x):
        return BooleanQuery().add(TermQuery(int(x[0])), Occur.SHOULD).add(TermQuery(int(x[1])), Occur.SHOULD)

    workloads = {
        "a_match_in_bool": [BooleanQuery().add(match(x), Occur.MUST).add(price, Occur.FILTER) for x in t],
        "c_multi_match_tie0.3": [BooleanQuery().add(DisjunctionMaxQuery([match(x), match(y)], 0.3), Occur.MUST).add(price, Occur.FILTER)
                                 for x, y in zip(t, u)],
    }
    terms = TermsCollector(CAT, 10, nested=(("top", TopHitsCollector(3)),))
    legs = {"terms": [terms], "filter": [terms, FilterCollector(fprice, (("t", terms),))]}

    ctx = GpuContext(0)
    whole = GpuIndex(ctx, sh)
    cuts = np.linspace(0, n, a.leaves + 1).astype(np.int64)
    cuts[1:-1] += 4099   # cut inside a window
    leaves = [GpuIndex(ctx, sh.doc_range(int(lo), int(hi))) for lo, hi in zip(cuts, cuts[1:])]
    targets = {"one_image": GpuIndexSearcher(whole), f"{a.leaves}_leaves": GpuLeafSearcher(ctx, leaves)}
    gpu = card()
    oix = oracle.OracleIndex(sh)
    sample = list(range(0, nq, max(1, nq // a.sample)))[:a.sample]
    tspec = {"top": ("top_hits", 3, 0)}

    def check_terms(o, q, want, what):
        m = want["n"]
        if not (o["n"][q] == m and o["keys"][q].tolist() == want["keys"].tolist() and o["counts"][q].tolist() == want["counts"].tolist()):
            raise SystemExit(f"{what}: buckets differ from the reference")
        for i in range(m):
            d, s_, tot = want["nested"]["top"][i]
            r = o["nested"]["top"]
            if not (r["counts"][q, i] == len(d) and r["total_hits"][q, i] == tot and r["docs"][q, i, :len(d)].tolist() == d.tolist()
                    and np.array_equal(r["scores"][q, i, :len(d)].view(np.uint32), s_.view(np.uint32))):
                raise SystemExit(f"{what}: top hits of slot {i} differ from the reference")

    refs = {}   # the sample's match sets and scores, per workload

    def gate(name, s, queries, leg):
        sub = [queries[i] for i in sample]
        if id(queries) not in refs:
            refs[id(queries)] = rtr.evaluate_all(sh, sub, oix)
        present, score = refs[id(queries)]
        res, outs = s.search_tree_with_collectors(sub, RelevanceCollector(k, INT_MAX), legs[leg])
        carr, _, qarr, _ = compile_queries([fprice])
        fmask = far.query_mask(oix, carr, qarr, 0)
        for i in range(len(sub)):
            if res.total_hits[i] != present[i].sum():
                raise SystemExit(f"{name}: totalHits differ from the reference (query {sample[i]})")
            check_terms(outs[0], i, nr.terms_nested(sh, present[i], CAT, 10, True, tspec, None, score[i]), f"{name} query {sample[i]}")
            if leg == "filter":
                sel = present[i] & fmask
                want = far.filter_result(sh, sel, {"t": ("terms", CAT, 10, True, tspec, None)}, score[i])
                if outs[1]["doc_count"][i] != want["doc_count"]:
                    raise SystemExit(f"{name}: docCount differs from the reference (query {sample[i]})")
                check_terms(outs[1]["t"], i, want["t"], f"{name} filter query {sample[i]}")

    def timed(run):
        for _ in range(a.warmup):
            run()
        ts = []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            run()
            ts.append((time.perf_counter() - t0) * 1e3)
        return {"median_ms": round(float(np.median(ts)), 2), "min_ms": round(float(np.min(ts)), 2)}

    for wname, queries in workloads.items():
        for tname, s in targets.items():
            for leg in legs:
                gate(f"{wname}/{tname}/{leg}", s, queries, leg)
            out = {"workload": wname, "target": tname, "docs": n, "batch": nq, "top_k": k, "gpu": gpu,
                   "unit": "ms per batch, host clock around a call that ends with its results on the host"}
            out["plain"] = timed(lambda: s.search_tree(queries, RelevanceCollector(k, INT_MAX)))
            for leg, adds in legs.items():
                out[leg] = timed(lambda: s.search_tree_with_collectors(queries, RelevanceCollector(k, INT_MAX), adds))
            print(json.dumps(out), flush=True)
    targets[f"{a.leaves}_leaves"].close()
    for x in leaves + [whole]:
        x.close()
    ctx.close()


if __name__ == "__main__":
    main()
