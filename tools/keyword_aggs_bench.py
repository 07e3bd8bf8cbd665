"""Batch time of terms aggregations over keyword columns against numeric terms aggregations of equal cardinality, on
bench.py's BM25 shape: 10M docs, 1024 3-term disjunctions per batch, terms size 10.

Keyword columns: a SORTED_SET column of 1-4 distinct terms per doc drawn Zipf(1.3) from 1,000, and a SORTED column of
20,000 terms. The numeric legs count an int column folded to 1,000 and to
20,000 distinct values. The legs are alternated step by step in one run, so they share the card's state. Each timed call is
one search_with_collectors over the whole batch: CUDA events on the default stream around it, and a host clock around the
same call, which ends with its results (keyword keys as str) on the host. The call is synchronous, so the event interval
spans its host work too (compiling, the selection copies, turning ordinals into str), not device time alone. Prints one JSON line with the median and min of
each leg and the card's name and power limit, read in the same run."""
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
from nrtsearch_b200.index import KeywordColumn  # noqa: E402
from nrtsearch_b200.search import (BooleanQuery, GpuContext, GpuIndex, GpuIndexSearcher, Occur, RelevanceCollector,  # noqa: E402
                                   TermQuery, TermsCollector)


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def sorted_set_column(n, n_terms, rng):
    """1-4 distinct Zipf-drawn ordinals per doc, ascending; terms "k00000" .. in byte order"""
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
        raise SystemExit("keyword_aggs_bench: no CUDA device")

    rng = np.random.default_rng(0x4B42)
    sh = ix.synth_text_shard(args.docs, args.vocab)
    col = ix.synth_int_column(args.docs)
    sh.columns = [col % 1000, col % 20_000]
    sh.column_has = [None, None]
    one = rng.integers(0, 20_000, args.docs).astype(np.int32)
    sh.keyword_columns = [sorted_set_column(args.docs, 1000, rng), KeywordColumn([b"s%05d" % i for i in range(20_000)], one)]
    terms = ix.synth_query_terms(args.nq, 3, args.vocab)
    queries = [BooleanQuery().add(TermQuery(int(t[0])), Occur.SHOULD).add(TermQuery(int(t[1])), Occur.SHOULD)
               .add(TermQuery(int(t[2])), Occur.SHOULD) for t in terms]
    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    coll = RelevanceCollector(args.topk)
    legs = {
        "keyword_sorted_set_1000": [TermsCollector(0, args.size, True, "keyword")],
        "numeric_1000": [TermsCollector(0, args.size, True, "int")],
        "keyword_sorted_20000": [TermsCollector(1, args.size, True, "keyword")],
        "numeric_20000": [TermsCollector(1, args.size, True, "int")],
    }
    values = int(sh.keyword_columns[0].offsets[-1])
    out = {"docs": args.docs, "nq": args.nq, "topk": args.topk, "size": args.size, "gpu": gpu_name(),
           "sorted_set_values_per_doc": round(values / args.docs, 3),
           "unit": "ms per batch: CUDA events around the whole synchronous call / host clock after its synchronise (both include "
                   "compile, upload and the host's key conversion)"}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, adds in legs.items():
        for _ in range(args.warmup):
            s.search_with_collectors(queries, coll, adds)
    dev = {name: [] for name in legs}
    host = {name: [] for name in legs}
    for _ in range(args.steps):   # legs alternated step by step
        for name, adds in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ev0.record()
            s.search_with_collectors(queries, coll, adds)
            ev1.record()
            torch.cuda.synchronize()
            host[name].append((time.perf_counter() - t0) * 1e3)
            dev[name].append(ev0.elapsed_time(ev1))
    for name in legs:
        out[name] = {"device_median_ms": round(float(np.median(dev[name])), 3), "device_min_ms": round(float(np.min(dev[name])), 3),
                     "host_median_ms": round(float(np.median(host[name])), 3), "host_min_ms": round(float(np.min(host[name])), 3)}
    print(json.dumps(out))
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
