"""ctypes binding of the test-only sort code harness (tests/csrc/sort_code_harness.cu) and the numpy restatement of what it
computes. The harness runs the product's sort_codes_build (the index-time codes of one column) and sort_code_of (the code
of an arbitrary value) on host arrays, so a test sees the codes that the sorted search hides behind its pages."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libsort_code_harness.so")
_lib = None
INVALID = 1
_SIGN = np.uint64(1 << 63)


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.sh_last_error.restype = C.c_char_p
        P, I = C.c_void_p, C.c_int32
        h.sh_codes.argtypes = [P, P, P, I, P, P, P]
        h.sh_code_of.argtypes = [P, I, P, I, P]
        _lib = h
    return _lib


class HarnessError(RuntimeError):
    def __init__(self, rc: int, msg: str):
        super().__init__(f"sort code harness status {rc}: {msg}")
        self.rc = rc


def _check(rc: int) -> None:
    if rc != 0:
        raise HarnessError(rc, lib().sh_last_error().decode("utf-8", "replace"))


def _ptr(a):
    return None if a is None else a.ctypes.data


def codes(values, has=None, int32: bool = False):
    """sort_codes_build over one column: (codes uint32[n], distinct uint64[n_distinct] sortable keys). int32 picks the
    int32 column layout of nrtgpu_index_build (a column whose values all fit), else int64."""
    v = np.ascontiguousarray(values, np.int32 if int32 else np.int64)
    n = len(v)
    h = None if has is None else np.ascontiguousarray(has, np.uint8)
    out = np.zeros(n, np.uint32)
    dist = np.zeros(max(n, 1), np.uint64)
    nd = C.c_int32(-1)
    _check(lib().sh_codes(None if int32 else _ptr(v), _ptr(v) if int32 else None, _ptr(h), n, out.ctypes.data, dist.ctypes.data,
                          C.byref(nd)))
    return out, dist[:nd.value].copy()


def code_of(distinct, probes):
    """sort_code_of of every probe value against the sorted distinct keys: uint32[len(probes)]"""
    d = np.ascontiguousarray(distinct, np.uint64)
    p = np.ascontiguousarray(probes, np.int64)
    out = np.zeros(len(p), np.uint32)
    _check(lib().sh_code_of(_ptr(d) if len(d) else None, len(d), _ptr(p), len(p), out.ctypes.data))
    return out


def sortable(values) -> np.ndarray:
    """the uint64 keys the codes are built over: the int64 value with its sign bit flipped"""
    return np.asarray(values, np.int64).view(np.uint64) ^ _SIGN


def reference_codes(values, has=None):
    """codes = 2 * searchsorted(unique(v), v) + 2 over the docs with a value, 0 for the others; the distinct keys"""
    v = np.asarray(values, np.int64)
    h = np.ones(len(v), bool) if has is None else np.asarray(has) != 0
    keys = np.unique(sortable(v[h]))
    out = np.zeros(len(v), np.uint32)
    out[h] = 2 * np.searchsorted(keys, sortable(v[h])) + 2
    return out, keys


def reference_code_of(distinct, probes):
    """2i + 2 when the probe is distinct value i, else 2i + 1 with i = the number of distinct values below it"""
    d = np.asarray(distinct, np.uint64)
    k = sortable(probes)
    i = np.searchsorted(d, k)
    hit = (i < len(d)) & (d[np.minimum(i, max(len(d) - 1, 0))] == k) if len(d) else np.zeros(len(k), bool)
    return np.where(hit, 2 * i + 2, 2 * i + 1).astype(np.uint32)
