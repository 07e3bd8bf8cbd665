"""Batch time of a terms aggregation alone, with a nested max, and with nested top hits, on bench.py's BM25 shape.

The shard is bench.py's synthetic corpus (10M docs, 1M terms by default) with one int column folded to 1000 distinct values
(bench.py's column has about a million, whose per-query count table would not fit a 1024-query batch); the queries are
bench.py's 3-term disjunctions. Each timed call is one search_with_collectors over the whole batch, host clock around a call
that ends with its results copied to the host, so it includes compiling and uploading the batch. Prints one JSON line
with the median and min of each leg and the GPU it ran on."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from nrtsearch_b200 import index as ix  # noqa: E402
from nrtsearch_b200.search import (BooleanQuery, GpuContext, GpuIndex, GpuIndexSearcher, MaxCollector, Occur,  # noqa: E402
                                   RelevanceCollector, TermQuery, TermsCollector, TopHitsCollector)


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--topk", type=int, default=100)
    ap.add_argument("--size", type=int, default=10, help="buckets returned")
    ap.add_argument("--top-hits", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()

    sh = ix.synth_text_shard(args.docs, args.vocab)
    col = ix.synth_int_column(args.docs)
    sh.columns = [col % 1000, col]
    sh.column_has = [None, None]
    terms = ix.synth_query_terms(args.nq, 3, args.vocab)
    queries = [BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD).add(TermQuery(int(t[1])), Occur.SHOULD)
               .add(TermQuery(int(t[2])), Occur.SHOULD) for t in terms]
    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    coll = RelevanceCollector(args.topk)
    legs = {
        "terms": TermsCollector(0, args.size, True, "int"),
        "terms_nested_max": TermsCollector(0, args.size, True, "int", (("max", MaxCollector(1, "int")),)),
        "terms_nested_top_hits": TermsCollector(0, args.size, True, "int", (("hits", TopHitsCollector(args.top_hits)),)),
    }
    out = {"docs": args.docs, "nq": args.nq, "topk": args.topk, "size": args.size, "top_hits": args.top_hits,
           "gpu": gpu_name(), "unit": "ms per batch (host clock, includes compile and upload)"}
    for name, a in legs.items():
        for _ in range(args.warmup):
            s.search_with_collectors(queries, coll, [a])
        t = []
        for _ in range(args.steps):
            t0 = time.perf_counter()
            s.search_with_collectors(queries, coll, [a])
            t.append((time.perf_counter() - t0) * 1e3)
        out[name] = {"median_ms": round(float(np.median(t)), 3), "min_ms": round(float(np.min(t)), 3)}
    print(json.dumps(out))
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
