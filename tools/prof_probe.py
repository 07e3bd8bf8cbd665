#!/usr/bin/env python
"""Launch sequence for ncu captures of the posting traversal kernels on the full-size workloads (BASELINE.json
configs[1] and configs[2]): N runs of the TOP_SCORES batch, N of the ScoreMode.COMPLETE batch, N of the conjunctive
batch -- nothing else launches a posting_probe kernel, so `ncu -k regex:posting_probe -s <skip> -c <count>` picks
launches by position. Without ncu it prints the CUDA-event kernel time of each leg (stage 0 of nrtgpu_batch_stage_ms).
With NRTGPU_DEBUG_MODES=1 the profiling instantiation writes its counters to stderr after every run: per item cycles,
runs, rounds, driver postings, flushes, and (pure disjunctions) the items that started without a threshold and those
whose MAXSCORE roles went stale.

  python tools/prof_probe.py [--runs 2] [--docs 10000000] [--legs top,complete,conj]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--topk", type=int, default=100)
    ap.add_argument("--legs", default="top,complete,conj")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build_if_needed()
    import bench
    from nrtsearch_b200 import index as ix
    from nrtsearch_b200.search import GpuContext, GpuIndex, GpuIndexSearcher, RelevanceCollector
    sh = ix.synth_text_shard(args.docs, args.vocab)
    sh.term_df = np.diff(sh.term_off).astype(np.int64)
    sh.columns = [ix.synth_int_column(args.docs)]
    sh.column_has = [None]
    ctx = GpuContext(0)
    gix = GpuIndex(ctx, sh)
    s = GpuIndexSearcher(gix)
    disj = bench.make_queries(args.nq, args.vocab)
    conj = bench.make_conj_queries(args.nq, args.vocab)
    out = {}
    for leg in args.legs.split(","):
        qs, thr = {"top": (disj, 1000), "complete": (disj, 2**31 - 1), "conj": (conj, 1000)}[leg]
        b = s.prepare(qs, RelevanceCollector(args.topk, thr))
        for _ in range(args.runs):
            b.run()
        import torch
        torch.cuda.synchronize()
        b.reset_timing()
        b.run()
        torch.cuda.synchronize()
        out[leg] = {"kernel_ms": b.stage_ms(0), "merge_ms": b.stage_ms(1), **b.stats()}
        b.close()
    print(json.dumps(out))
    gix.close()
    ctx.close()


if __name__ == "__main__":
    main()
