"""Batch time of nested top hits by score and by a Sort, on one image and over leaves, on tools/nested_aggs_bench.py's batch.

The shard is bench.py's synthetic corpus (10M docs, 1M terms by default) with one int column folded to 1000 distinct values
for the terms buckets, the column itself and a second int column for the Sorts; the queries are bench.py's 3-term
disjunctions; each call carries one terms aggregation (size 10) with one nested top-5. Legs: top hits by score, by a
one-field Sort and by a three-field Sort (a column, a second column descending, the doc id), each on one image and on
--leaves doc-range leaves of a GpuLeafSearcher. The Sorts' orders are built before timing (GpuIndex.sort_order caches them).
Each timed call is one search_with_collectors over the whole batch, host clock around a call that ends with its results
copied to the host, so it includes compiling and uploading the batch. Prints one JSON line with the median and min of each
leg and the GPU it ran on, with its power limit."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from nested_aggs_bench import gpu_name  # noqa: E402
from nrtsearch_b200 import index as ix  # noqa: E402
from nrtsearch_b200.search import (BooleanQuery, GpuContext, GpuIndex, GpuIndexSearcher, GpuLeafSearcher, Occur,  # noqa: E402
                                   RelevanceCollector, SortType, TermQuery, TermsCollector, TopHitsCollector)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--topk", type=int, default=100)
    ap.add_argument("--size", type=int, default=10, help="buckets returned")
    ap.add_argument("--top-hits", type=int, default=5)
    ap.add_argument("--leaves", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    sh = ix.synth_text_shard(args.docs, args.vocab)
    col = ix.synth_int_column(args.docs)
    sh.columns = [col % 1000, col, (col * 2654435761) % 100_003]
    sh.column_has = [None, None, None]
    terms = ix.synth_query_terms(args.nq, 3, args.vocab)
    queries = [BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD).add(TermQuery(int(t[1])), Occur.SHOULD)
               .add(TermQuery(int(t[2])), Occur.SHOULD) for t in terms]
    ctx = GpuContext(0)
    whole = GpuIndex(ctx, sh)
    cuts = np.linspace(0, args.docs, args.leaves + 1).astype(np.int64)
    leaves = [GpuIndex(ctx, sh.doc_range(int(a), int(b))) for a, b in zip(cuts, cuts[1:])]
    targets = {"one_image": GpuIndexSearcher(whole), f"{args.leaves}_leaves": GpuLeafSearcher(ctx, leaves)}
    sorts = {"score": None, "sort_1_field": [SortType(1, field_type="int")],
             "sort_3_fields": [SortType(2, field_type="int"), SortType(1, True, field_type="int"), SortType("docid")]}
    coll = RelevanceCollector(args.topk)
    out = {"docs": args.docs, "nq": args.nq, "topk": args.topk, "size": args.size, "top_hits": args.top_hits,
           "leaves": args.leaves, "gpu": gpu_name(), "unit": "ms per batch (host clock, includes compile and upload)"}
    for tname, s in targets.items():
        for sname, sort in sorts.items():
            a = TermsCollector(0, args.size, True, "int", (("hits", TopHitsCollector(args.top_hits, 0, sort)),))
            for _ in range(args.warmup):
                s.search_with_collectors(queries, coll, [a])
            t = []
            for _ in range(args.steps):
                t0 = time.perf_counter()
                s.search_with_collectors(queries, coll, [a])
                t.append((time.perf_counter() - t0) * 1e3)
            out[f"{tname}/{sname}"] = {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(np.min(t)), 3)}
    print(json.dumps(out))
    targets[f"{args.leaves}_leaves"].close()
    for g in leaves + [whole]:
        g.close()
    ctx.close()


if __name__ == "__main__":
    main()
