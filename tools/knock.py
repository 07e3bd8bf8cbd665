#!/usr/bin/env python
"""Knock-out timing of the posting kernel (profiling aid): one index build, then the TOP_SCORES / COMPLETE / conj batches
timed with parts of the kernel disabled through NRTGPU_KNOCK (results are wrong by construction; only times matter).
Needs a library built with -DNRT_PROBE_KNOCK (make EXTRA=-DNRT_PROBE_KNOCK in nrtsearch_b200/csrc, or a variant build
loaded through NRTGPU_LIB_PATH): the production build compiles the switches out."""
import json, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g
g.build_if_needed()
import bench
import torch
from nrtsearch_b200 import index as ix
from nrtsearch_b200.search import GpuContext, GpuIndex, GpuIndexSearcher, RelevanceCollector
docs = int(sys.argv[1]) if len(sys.argv) > 1 else 10_000_000
knocks = [int(x) for x in (sys.argv[2] if len(sys.argv) > 2 else "0,1,2,4,3,7,8,24").split(",")]
sh = ix.synth_text_shard(docs, 1_000_000)
sh.term_df = np.diff(sh.term_off).astype(np.int64)
sh.columns = [ix.synth_int_column(docs)]; sh.column_has = [None]
ctx = GpuContext(0); gix = GpuIndex(ctx, sh); s = GpuIndexSearcher(gix)
disj = bench.make_queries(1024, 1_000_000); conj = bench.make_conj_queries(1024, 1_000_000)
for k in knocks:
    os.environ["NRTGPU_KNOCK"] = str(k)
    out = {}
    for leg, (qs, thr) in {"top": (disj, 1000), "complete": (disj, 2**31 - 1), "conj": (conj, 1000)}.items():
        b = s.prepare(qs, RelevanceCollector(100, thr))
        for _ in range(2): b.run()
        torch.cuda.synchronize(); b.reset_timing()
        for _ in range(3): b.run()
        torch.cuda.synchronize()
        out[leg] = round(b.stage_ms(0), 3)
        b.close()
    print("knock", k, json.dumps(out), flush=True)
