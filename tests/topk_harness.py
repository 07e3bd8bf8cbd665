"""ctypes binding of the test-only top-k harness (tests/csrc/topk_harness.cu). The harness runs the product's
merge_slices_kernel (the per-query merge of a batch's work-item lists) and flush_top_k (a posting kernel's candidate cut
and threshold publication) on host arrays, so a test can hold them against tests/topk_reference.py at any shape."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libtopk_harness.so")
_lib = None
INVALID = 1
SENTINEL = -7   # what the outputs hold before a call


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.th_last_error.restype = C.c_char_p
        P, I = C.c_void_p, C.c_int32
        h.th_merge_slices.argtypes = [I, I, I, I, P, P, P, P, P, P, C.c_longlong, P, P, P, P, P, P]
        h.th_flush_top_k.argtypes = [I, I, P, P, I, C.c_uint64, P, P]
        _lib = h
    return _lib


class HarnessError(RuntimeError):
    def __init__(self, rc: int, msg: str):
        super().__init__(f"top-k harness status {rc}: {msg}")
        self.rc = rc


def _check(rc: int) -> None:
    if rc != 0:
        raise HarnessError(rc, lib().th_last_error().decode("utf-8", "replace"))


def _in(a, dtype):
    return None if a is None else np.ascontiguousarray(a, dtype)


def _ptr(a):
    return None if a is None else a.ctypes.data



def merge_slices(keys, counts, top_k: int, doc_base: int = 0, theta=None, total_hits=None, pruned=None, terminated=None,
                 terminate_after: int = 0, known_hits=None, want_total: bool = False, want_flags: bool = False):
    """merge_slices_kernel over keys uint64 [nq, n_lists, top_k] with counts [nq, n_lists]. Optional inputs are [nq] arrays
    or None (absent). The outputs start as SENTINEL words, so slots the kernel does not write keep it. Returns a dict:
    docs [nq, top_k], scores [nq, top_k], counts [nq], terminated [nq] or None, total [nq] or None, flags [nq] or None."""
    k = np.ascontiguousarray(keys, np.uint64)
    c = np.ascontiguousarray(counts, np.int32)
    nq, n_lists = c.shape
    assert k.shape == (nq, n_lists, top_k)
    docs = np.full((nq, top_k), SENTINEL, np.int32)
    scores = np.full((nq, top_k), SENTINEL, np.int32).view(np.float32)
    out_counts = np.full(nq, SENTINEL, np.int32)
    term = _in(terminated, np.int32)
    term = None if term is None else term.copy()
    total = np.full(nq, SENTINEL, np.int64) if want_total else None
    flags = np.full(nq, SENTINEL, np.int32) if want_flags else None
    th, tot, pr, kn = _in(theta, np.uint64), _in(total_hits, np.uint64), _in(pruned, np.int32), _in(known_hits, np.uint64)
    _check(lib().th_merge_slices(nq, n_lists, top_k, doc_base, _ptr(k), _ptr(c), _ptr(th), _ptr(tot), _ptr(pr), _ptr(term),
                                 int(terminate_after), _ptr(kn), _ptr(docs), _ptr(scores), _ptr(out_counts), _ptr(total),
                                 _ptr(flags)))
    return {"docs": docs, "scores": scores, "counts": out_counts, "terminated": term, "total": total, "flags": flags}


def flush_top_k(cand, count: int, cap: int, top_k: int, dec: int, g_theta: int, theta: int, n_threads: int):
    """flush_top_k in one CTA of n_threads: cand uint64 [cap] holding `count` keys. Returns (cand after the flush, count,
    g_theta, theta)."""
    buf = np.ascontiguousarray(cand, np.uint64).copy()
    assert buf.shape == (cap,)
    n, g, t = C.c_int32(count), C.c_uint64(g_theta), C.c_uint64(theta)
    _check(lib().th_flush_top_k(cap, n_threads, buf.ctypes.data, C.byref(n), top_k, dec, C.byref(g), C.byref(t)))
    return buf, n.value, g.value, t.value
