"""Batch time of filter collectors on bench.py's BM25 shape: a terms aggregation alone, the same terms aggregation under a
query filter, under a value-set filter, and a filter with nested top 5 hits.

The shard is bench.py's synthetic corpus (10M docs, 1M terms by default) with an int column folded to 1000 distinct values
(the terms column) and one folded to 100 (the value-set column); the queries are bench.py's 3-term disjunctions, 1024 per
batch. The query filter is a disjunction of a dense term and a range on the terms column; the value set holds 10 of the
100 values. Each timed call is one search_with_collectors over the whole batch: CUDA events on the default stream around
it, and a host clock around the same call, which ends with its results copied to the host (so it includes compiling,
uploading and building the filter rows). Prints one JSON line with the median and min of each leg and the card's name
and power limit."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from nrtsearch_b200 import index as ix  # noqa: E402
from nrtsearch_b200.search import (BooleanQuery, FilterCollector, GpuContext, GpuIndex, GpuIndexSearcher, Occur,  # noqa: E402
                                   RangeQuery, RelevanceCollector, TermQuery, TermsCollector, TopHitsCollector, ValueSetFilter)


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
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("filter_aggs_bench: no CUDA device")

    sh = ix.synth_text_shard(args.docs, args.vocab)
    col = ix.synth_int_column(args.docs)
    sh.columns = [col % 1000, col % 100]
    sh.column_has = [None, None]
    terms = ix.synth_query_terms(args.nq, 3, args.vocab)
    queries = [BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD).add(TermQuery(int(t[1])), Occur.SHOULD)
               .add(TermQuery(int(t[2])), Occur.SHOULD) for t in terms]
    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    coll = RelevanceCollector(args.topk)
    t = TermsCollector(0, args.size, True, "int")
    qfilter = BooleanQuery().add(TermQuery(0), Occur.SHOULD).add(RangeQuery(0, 0, 499), Occur.SHOULD)
    vset = ValueSetFilter(1, tuple(range(0, 100, 10)), "int")
    legs = {
        "terms": [t],
        "terms_under_query_filter": [FilterCollector(qfilter, (("t", t),))],
        "terms_under_value_set": [FilterCollector(vset, (("t", t),))],
        "filter_nested_top_hits": [FilterCollector(qfilter, (("hits", TopHitsCollector(5)),))],
    }
    out = {"docs": args.docs, "nq": args.nq, "topk": args.topk, "size": args.size, "gpu": gpu_name(),
           "unit": "ms per batch: device events / host clock after the call's synchronise (both include compile and upload)"}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, adds in legs.items():
        for _ in range(args.warmup):
            s.search_with_collectors(queries, coll, adds)
        dev, host = [], []
        for _ in range(args.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ev0.record()
            s.search_with_collectors(queries, coll, adds)
            ev1.record()
            torch.cuda.synchronize()
            host.append((time.perf_counter() - t0) * 1e3)
            dev.append(ev0.elapsed_time(ev1))
        out[name] = {"device_median_ms": round(float(np.median(dev)), 3), "device_min_ms": round(float(np.min(dev)), 3),
                     "host_median_ms": round(float(np.median(host)), 3), "host_min_ms": round(float(np.min(host)), 3)}
    print(json.dumps(out))
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
