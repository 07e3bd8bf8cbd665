"""Doc-range sharding across GPUs (SURVEY.md 8e): one shard group per GPU, one process per GPU.

Shard g holds global docs [g*N/G, (g+1)*N/G) with docBase = g*N/G -- exactly how Lucene leaves compose
global ids (reference src/main/java/org/apache/lucene/search/LazyQueueTopScoreDocCollector.java:74,148) --
plus a REPLICATED copy of the index-wide statistics (docFreq, docCount, sumTotalTermFreq), so idf and avgdl
are identical on every shard. A search step is: local top-k on every rank -> ONE all-gather of
[nq, k] x (doc, score) + [nq] counts -> TopDocs.merge on every rank
(reference .../LazyQueueTopScoreDocCollectorManager.java:137-144). torch.distributed is plumbing only.
"""
from __future__ import annotations

from typing import Tuple

import numpy as np

from .index import HostShard


def shard_range(n_docs: int, rank: int, world: int) -> Tuple[int, int]:
    return n_docs * rank // world, n_docs * (rank + 1) // world


def install_global_stats(shard: HostShard, device=None, group=None) -> HostShard:
    """All-reduce per-shard term statistics once at build time (NCCL on GPU tensors, gloo on CPU tensors)."""
    import torch
    import torch.distributed as dist
    local_df = np.diff(shard.term_off).astype(np.int64)
    nf = len(shard.fields)
    tail = np.array([x for f in shard.fields for x in (f.sum_total_term_freq, f.doc_count)], np.int64)
    t = torch.from_numpy(np.concatenate([local_df, tail]))
    if device is not None:
        t = t.to(device)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, group=group)
    g = t.cpu().numpy()
    shard.term_df = np.ascontiguousarray(g[:len(local_df)])
    for i, f in enumerate(shard.fields):
        f.sum_total_term_freq = int(g[len(local_df) + 2 * i])
        f.doc_count = int(g[len(local_df) + 2 * i + 1])
    assert nf == len(shard.fields)
    return shard


class TopKGather:
    """Pre-allocated buffers for the per-step all-gather of the local top-k (device or CPU tensors)."""

    def __init__(self, nq: int, k: int, world: int, device):
        import torch
        self.nq, self.k, self.world = nq, k, world
        self.loc_docs = torch.zeros(nq * k, dtype=torch.int32, device=device)
        self.loc_scores = torch.zeros(nq * k, dtype=torch.float32, device=device)
        self.loc_counts = torch.zeros(nq, dtype=torch.int32, device=device)
        self.all_docs = torch.zeros(world * nq * k, dtype=torch.int32, device=device)
        self.all_scores = torch.zeros(world * nq * k, dtype=torch.float32, device=device)
        self.all_counts = torch.zeros(world * nq, dtype=torch.int32, device=device)
        self.fin_docs = torch.zeros(nq * k, dtype=torch.int32, device=device)
        self.fin_scores = torch.zeros(nq * k, dtype=torch.float32, device=device)
        self.fin_counts = torch.zeros(nq, dtype=torch.int32, device=device)

    def gather(self, group=None):
        import torch.distributed as dist
        if self.world == 1:
            self.all_docs.copy_(self.loc_docs); self.all_scores.copy_(self.loc_scores); self.all_counts.copy_(self.loc_counts)
            return
        dist.all_gather_into_tensor(self.all_docs, self.loc_docs, group=group)
        dist.all_gather_into_tensor(self.all_scores, self.loc_scores, group=group)
        dist.all_gather_into_tensor(self.all_counts, self.loc_counts, group=group)

    def merge_on_device(self, ctx, stream: int):
        """TopDocs.merge of the gathered lists by the CUDA merge kernel (nrtgpu_merge_topk_device)."""
        import ctypes
        from . import _native
        _native.check(_native.gpu_lib().nrtgpu_merge_topk_device(
            ctx.handle, self.world, self.nq, self.k, self.all_docs.data_ptr(), self.all_scores.data_ptr(),
            self.all_counts.data_ptr(), self.fin_docs.data_ptr(), self.fin_scores.data_ptr(), self.fin_counts.data_ptr(),
            ctypes.c_void_p(stream)))


class PackedGather:
    """The ONE exchange step of a multi-GPU search (SURVEY.md 8e): every rank's packed result record
    (docs, scores, counts, relation flags, totalHits of all queries; include/nrtgpu.h nrtgpu_packed_words) is
    all-gathered once, then nrtgpu_merge_topk_packed does TopDocs.merge on every rank. Results never leave the device
    between the shard search and the merged page."""

    def __init__(self, nq: int, k: int, world: int, device):
        import torch
        from . import _native
        self.nq, self.k, self.world = nq, k, world
        self.words = int(_native.gpu_lib().nrtgpu_packed_words(nq, k)) if device.type == "cuda" else packed_words(nq, k)
        self.local = torch.zeros(self.words, dtype=torch.int32, device=device)
        self.all = torch.zeros(world * self.words, dtype=torch.int32, device=device)
        self.merged = torch.zeros(self.words, dtype=torch.int32, device=device)

    def gather(self, group=None):
        import torch.distributed as dist
        if self.world == 1:
            self.all.copy_(self.local)
        else:
            dist.all_gather_into_tensor(self.all, self.local, group=group)

    def merge_on_device(self, ctx, stream: int):
        import ctypes
        from . import _native
        _native.check(_native.gpu_lib().nrtgpu_merge_topk_packed(
            ctx.handle, self.world, self.nq, self.k, self.all.data_ptr(), self.merged.data_ptr(), ctypes.c_void_p(stream)))

    def unpack(self, record=None):
        """Host view of a record: docs [nq,k], scores [nq,k], counts [nq], flags [nq], total_hits [nq]."""
        r = (self.merged if record is None else record).cpu().numpy()
        return unpack_record(r, self.nq, self.k)


class SortedPackedGather:
    """The sorted counterpart of PackedGather: every rank's packed sorted record (docs, counts, flags, totalHits and the
    FieldDoc values of all queries; include/nrtgpu.h nrtgpu_sorted_packed_words), filled by
    nrtgpu_search_sorted_fields_packed, is all-gathered once, then nrtgpu_merge_sorted_packed does TopFieldDocs.merge on
    every rank. fields: the Sort's SortTypes (search.SortType). A Sort with a keyword field is refused: its values are
    codes of each shard's own term dictionary, which do not compare across shards."""

    def __init__(self, nq: int, k: int, fields, world: int, device):
        import torch
        from . import _native
        self.nq, self.k, self.world = nq, k, world
        self.fields = list(fields)
        if any(getattr(f, "field_type", None) == "keyword" and f.field not in ("docid", "score") for f in self.fields):
            raise _native.NrtGpuUnsupported(3, "a Sort with a keyword field does not merge across shards: each shard numbers "
                                               "its own term dictionary")
        self.n_fields = len(self.fields)
        self.words = (int(_native.gpu_lib().nrtgpu_sorted_packed_words(nq, k, self.n_fields)) if device.type == "cuda"
                      else sorted_packed_words(nq, k, self.n_fields))
        self.local = torch.zeros(self.words, dtype=torch.int32, device=device)
        self.all = torch.zeros(world * self.words, dtype=torch.int32, device=device)
        self.merged = torch.zeros(self.words, dtype=torch.int32, device=device)

    def gather(self, group=None):
        import torch.distributed as dist
        if self.world == 1:
            self.all.copy_(self.local)
        else:
            dist.all_gather_into_tensor(self.all, self.local, group=group)

    def merge_on_device(self, ctx, stream: int):
        import ctypes
        from . import _native
        cf = [f.c_field() for f in self.fields]
        arr = (_native.SortField * len(cf))(*cf)
        _native.check(_native.gpu_lib().nrtgpu_merge_sorted_packed(
            ctx.handle, arr, self.n_fields, self.world, self.nq, self.k, self.all.data_ptr(), self.merged.data_ptr(),
            ctypes.c_void_p(stream)))

    def unpack(self, record=None):
        """Host view of a record: docs [nq,k], values [nq,k,n_fields], counts [nq], flags [nq], total_hits [nq]."""
        r = (self.merged if record is None else record).cpu().numpy()
        return unpack_sorted_record(r, self.nq, self.k, self.n_fields)


def sorted_packed_words(nq: int, k: int, n_fields: int) -> int:
    w = (nq * k + 2 * nq + 1) & ~1
    return w + 2 * nq + 2 * nq * k * n_fields


def unpack_sorted_record(r: np.ndarray, nq: int, k: int, n_fields: int):
    n = nq * k
    w = (n + 2 * nq + 1) & ~1
    docs = r[:n].reshape(nq, k)
    counts = r[n:n + nq]
    flags = r[n + nq:n + 2 * nq]
    total = r[w:w + 2 * nq].view(np.int64)
    values = r[w + 2 * nq:w + 2 * nq + 2 * n * n_fields].view(np.int64).reshape(nq, k, n_fields)
    return docs, values, counts, flags, total


def packed_words(nq: int, k: int) -> int:
    w = nq * k * 2 + 2 * nq
    w = (w + 1) & ~1
    return w + 2 * nq


def unpack_record(r: np.ndarray, nq: int, k: int):
    n = nq * k
    w = (2 * n + 2 * nq + 1) & ~1
    docs = r[:n].reshape(nq, k)
    scores = r[n:2 * n].view(np.float32).reshape(nq, k)
    counts = r[2 * n:2 * n + nq]
    flags = r[2 * n + nq:2 * n + 2 * nq]
    total = r[w:w + 2 * nq].view(np.int64)
    return docs, scores, counts, flags, total
