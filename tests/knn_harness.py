"""ctypes binding of the test-only kNN kernel harness (tests/csrc/knn_harness.cu) and the plain numpy restatements the
kernel tests compare it with. The harness launches the product's candidate-stage kernels directly, so a test sees the
approximate scores and the fused epilogue's survivors that the end-to-end path hides behind the exact re-score."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libknn_harness.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.kh_last_error.restype = C.c_char_p
        h.kh_f32_to_bf16.argtypes = [C.c_void_p, C.c_void_p, C.c_int64]
        h.kh_gemm_bf16.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                   C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        h.kh_dot_tile.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
        _lib = h
    return _lib


def _check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError(f"knn harness status {rc}: {lib().kh_last_error().decode('utf-8', 'replace')}")


def _ptr(a):
    return None if a is None else a.ctypes.data


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def device_bf16(x: np.ndarray) -> np.ndarray:
    """The product's fp32 -> bf16 conversion (tc::f32_to_bf16_kernel), widened back to float32."""
    x = _f32(x)
    out = np.empty(x.shape, np.uint16)
    _check(lib().kh_f32_to_bf16(x.ctypes.data, out.ctypes.data, x.size))
    return (out.astype(np.uint32) << 16).view(np.float32)


def gemm_scores(Q, D, sim: int, n_base: int = 0, N: int = None) -> np.ndarray:
    """Unfused knn_gemm_bf16_kernel: approximate scores [M][N] of corpus rows [n_base, n_base + N) of D."""
    Q, D = _f32(Q), _f32(D)
    N = D.shape[0] - n_base if N is None else N
    S = np.empty((Q.shape[0], N), np.float32)
    _check(lib().kh_gemm_bf16(Q.ctypes.data, Q.shape[0], D.ctypes.data, D.shape[0], D.shape[1], n_base, N, sim,
                              S.ctypes.data, None, None, 0, None, None, 0, None, None))
    return S


def gemm_fused(Q, D, sim: int, theta, cc_cap: int, n_base: int = 0, N: int = None, filter_docs=None, live_docs=None,
               vec_docs=None, n_docs: int = 0):
    """Fused knn_gemm_bf16_kernel: (survivor keys [M][cc_cap], survivor counts [M]). filter_docs / live_docs are per doc
    (uint8, n_docs), vec_docs maps every corpus ordinal to its doc."""
    Q, D = _f32(Q), _f32(D)
    M = Q.shape[0]
    N = D.shape[0] - n_base if N is None else N
    theta = _f32(theta)
    f = None if filter_docs is None else np.ascontiguousarray(filter_docs, np.uint8)
    lb = None if live_docs is None else live_bits(live_docs)
    vd = None if vec_docs is None else np.ascontiguousarray(vec_docs, np.int32)
    cc = np.zeros((M, cc_cap), np.uint64)
    cnt = np.zeros(M, np.int32)
    _check(lib().kh_gemm_bf16(Q.ctypes.data, M, D.ctypes.data, D.shape[0], D.shape[1], n_base, N, sim, None,
                              theta.ctypes.data, _ptr(f), n_docs, _ptr(lb), _ptr(vd), cc_cap, cc.ctypes.data, cnt.ctypes.data))
    return cc, cnt


def dot_tile_scores(Q, D, sim: int) -> np.ndarray:
    """knn_dot_tile_kernel (fp32 SIMT candidate stage): approximate scores [M][N]."""
    Q, D = _f32(Q), _f32(D)
    S = np.empty((Q.shape[0], D.shape[0]), np.float32)
    _check(lib().kh_dot_tile(Q.ctypes.data, Q.shape[0], D.ctypes.data, D.shape[0], D.shape[1], sim, S.ctypes.data))
    return S


# ---- plain references ----

def bf16_round(x) -> np.ndarray:
    """fp32 -> bf16 (round to nearest, ties to even), widened back to float32. Finite inputs only."""
    b = _f32(x).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32).reshape(np.shape(x))


def below_midpoint(rng, shape, exp_lo: int = -8, exp_hi: int = 1) -> np.ndarray:
    """Positive fp32 values a few fp32 ulps below the midpoint between a bf16 value with mantissa 1.0 or 1 + 2^-7 and its
    upper neighbour: each rounds DOWN to bf16 with relative error in (2^-8 / (1 + 2^-6), 2^-8). The exponent spread makes
    the fp32 sums of their products round as well."""
    e = rng.integers(exp_lo, exp_hi + 1, size=shape)
    mant = rng.integers(0, 2, size=shape)                       # 7-bit bf16 mantissa 0 or 1
    bf = ((e + 127).astype(np.uint32) << 7 | mant.astype(np.uint32)) << 16
    return (bf + 0x8000 - rng.integers(1, 16, size=shape).astype(np.uint32)).view(np.float32)


def make_key(score, ordinal) -> np.ndarray:
    """common.cuh make_key: ordered(score) << 32 | ~ordinal (keys order as (score desc, ordinal asc))."""
    b = _f32(score).view(np.uint32).astype(np.uint64)
    ordered = np.where(b & 0x80000000, ~b & 0xFFFFFFFF, b | 0x80000000)
    return (ordered << np.uint64(32)) | (~np.asarray(ordinal, np.uint64) & 0xFFFFFFFF)


def live_bits(live_docs) -> np.ndarray:
    """Per-doc 0/1 bytes -> the engine's liveDocs bitmap (bit d & 31 of word d >> 5)."""
    live = np.asarray(live_docs, np.uint8)
    words = np.zeros((len(live) + 31) // 32, np.uint32)
    d = np.nonzero(live)[0]
    np.bitwise_or.at(words, d >> 5, np.left_shift(np.uint32(1), (d & 31).astype(np.uint32)))
    return words


def approx_reference(Q, D, sim: int, norm2=None) -> np.ndarray:
    """float64 candidate score of every (query, vector) pair: dot / mip: <q, d>; cosine: <q, d> / |d|;
    l2: 2 <q, d> - |d|^2 (the per-query constant |q|^2 dropped, as in the kernels). norm2 defaults to |d|^2 of D."""
    Q, D = np.asarray(Q, np.float64), np.asarray(D, np.float64)
    dot = Q @ D.T
    n2 = (D * D).sum(axis=1) if norm2 is None else np.asarray(norm2, np.float64)
    if sim == 2:
        return dot / np.sqrt(np.maximum(n2, 1e-30))[None, :]
    if sim == 0:
        return 2.0 * dot - n2[None, :]
    return dot
