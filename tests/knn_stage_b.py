"""ctypes binding of the test-only harness of the kNN kernels that run after the candidate GEMM
(tests/csrc/knn_stage_b_harness.cu) and the plain numpy restatements their tests compare them with. The harness launches
the product's select, merge, re-score, exact-fallback and index-time kernels directly, so a test sees the candidate
lists, the certificate's decisions and the exact fallback's chunk lists that the end-to-end path hides behind the final
page. The candidate stage's launchers and helpers of tests/knn_harness.py are re-exported, so a test needs one import."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from knn_harness import (_f32, _ptr, approx_reference, below_midpoint, bf16_round, gemm_fused, gemm_scores,  # noqa: F401
                         live_bits, make_key)

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc", "libknn_stage_b_harness.so")
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            raise ImportError(f"{_PATH} is missing: build it with `make -C nrtsearch_b200/csrc`")
        h = C.CDLL(_PATH)
        h.kh_last_error.restype = C.c_char_p
        P, I = C.c_void_p, C.c_int
        h.kh_select.argtypes = [P, I, I, I, I, I, P, P, P, P, P, I, P, I, P, I, I, P]
        h.kh_merge_chunk.argtypes = [I, I, I, P, P, P, P, P, P]
        h.kh_rescore.argtypes = [P, I, P, I, I, I, P, P, I, I, P, I, P, C.c_float, C.c_float, P, P, P, P]
        h.kh_exact.argtypes = [P, I, P, I, I, I, P, I, I, I, P, P, P, I, P, I, P, I, I, P, P, C.c_int64, P, P, P, P, P, P, P]
        h.kh_prepare.argtypes = [P, I, I, I, P, P, P]
        _lib = h
    return _lib


def _check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError(f"knn harness status {rc}: {lib().kh_last_error().decode('utf-8', 'replace')}")


THETA_UNSET = np.float32(-12345.0)   # pre-fill of a threshold output: "the kernel did not write it" is observable
BYTE_FLAG = 0x100                    # kKnnByteFlag: byte-vector score mapping


def _i32(a):
    return None if a is None else np.ascontiguousarray(a, np.int32)


def _rows(row_bits, qrow):
    """(row bitmaps uint32[n_rows][words] or None, n_rows, words, qrow int32 or None)"""
    if qrow is None:
        return None, 0, 0, None
    r = np.ascontiguousarray(row_bits, np.uint32)
    return r, r.shape[0], r.shape[1], _i32(qrow)


def select(S, kprime: int, cand=None, cand_cnt=None, theta=None, chunk_base: int = 0, n_chunk: int = None, filter_docs=None,
           live_docs=None, n_docs: int = 0, vec_docs=None, row_bits=None, qrow=None):
    """knn_select_kernel over the score rows S[nq][ldS]: (cand uint64[nq][kprime], cand_cnt[nq], theta[nq]). cand /
    cand_cnt are the incoming lists (default: empty), theta the incoming threshold outputs (default: THETA_UNSET)."""
    S = _f32(S)
    nq, ldS = S.shape
    n_chunk = ldS if n_chunk is None else n_chunk
    cand = np.zeros((nq, kprime), np.uint64) if cand is None else np.ascontiguousarray(cand, np.uint64).copy()
    cnt = np.zeros(nq, np.int32) if cand_cnt is None else np.ascontiguousarray(cand_cnt, np.int32).copy()
    th = np.full(nq, THETA_UNSET, np.float32) if theta is None else _f32(theta).copy()
    assert cand.shape == (nq, kprime)
    f = None if filter_docs is None else np.ascontiguousarray(filter_docs, np.uint8)
    lb = None if live_docs is None else live_bits(live_docs)
    vd = _i32(vec_docs)
    rb, n_rows, words, qr = _rows(row_bits, qrow)
    _check(lib().kh_select(S.ctypes.data, nq, ldS, n_chunk, chunk_base, kprime, cand.ctypes.data, cnt.ctypes.data,
                           th.ctypes.data, _ptr(f), _ptr(lb), n_docs, _ptr(vd), 0 if vd is None else len(vd), _ptr(rb), n_rows,
                           words, _ptr(qr)))
    return cand, cnt, th


def merge_chunk(cand, cand_cnt, cc, cc_cnt, theta=None):
    """knn_merge_chunk_kernel: (cand, cand_cnt, theta, cc_cnt after, overflow flag)."""
    cand = np.ascontiguousarray(cand, np.uint64).copy()
    cc = np.ascontiguousarray(cc, np.uint64)
    nq, kprime = cand.shape
    cnt = np.ascontiguousarray(cand_cnt, np.int32).copy()
    ccn = np.ascontiguousarray(cc_cnt, np.int32).copy()
    th = np.full(nq, THETA_UNSET, np.float32) if theta is None else _f32(theta).copy()
    ovf = np.zeros(1, np.int32)
    _check(lib().kh_merge_chunk(nq, kprime, cc.shape[1], cand.ctypes.data, cnt.ctypes.data, cc.ctypes.data, ccn.ctypes.data,
                                th.ctypes.data, ovf.ctypes.data))
    return cand, cnt, th, ccn, int(ovf[0])


def rescore(Q, D, sim: int, cand, cand_cnt, k: int, eps_rel: float, dmax: float, vec_docs=None, doc_base: int = 0, boosts=None):
    """knn_rescore_kernel on the candidate lists cand[nq][kprime]: (docs [nq][k], scores, counts, unsafe)."""
    Q, D = _f32(Q), _f32(D)
    cand = np.ascontiguousarray(cand, np.uint64)
    nq, kprime = cand.shape
    cnt, vd = _i32(cand_cnt), _i32(vec_docs)
    b = None if boosts is None else _f32(boosts)
    docs, scores = np.zeros((nq, k), np.int32), np.zeros((nq, k), np.float32)
    counts, unsafe = np.zeros(nq, np.int32), np.zeros(nq, np.int32)
    _check(lib().kh_rescore(Q.ctypes.data, nq, D.ctypes.data, D.shape[0], D.shape[1], sim, cand.ctypes.data, cnt.ctypes.data,
                            kprime, k, _ptr(vd), doc_base, _ptr(b), eps_rel, dmax, docs.ctypes.data, scores.ctypes.data,
                            counts.ctypes.data, unsafe.ctypes.data))
    return docs, scores, counts, unsafe


EXACT_CHUNK = 4096   # kKnnExactChunk


def exact(Q, D, sim: int, k: int, qsel=None, boosts=None, filter_docs=None, live_docs=None, n_docs: int = None, vec_docs=None,
          doc_base: int = 0, row_bits=None, qrow=None, ord_lists=None):
    """knn_exact_chunk_kernel + merge_slices_kernel: (keys [n_sel][n_chunks][k], cnt [n_sel][n_chunks], docs [n_sel][k],
    scores, counts). ord_lists (gather mode): one ordinal list per filter row."""
    Q, D = _f32(Q), _f32(D)
    nq, n = Q.shape[0], D.shape[0]
    qsel = np.arange(nq, dtype=np.int32) if qsel is None else _i32(qsel)
    n_sel = len(qsel)
    n_docs = n if n_docs is None else n_docs
    b = None if boosts is None else _f32(boosts)
    f = None if filter_docs is None else np.ascontiguousarray(filter_docs, np.uint8)
    lb = None if live_docs is None else live_bits(live_docs)
    vd = _i32(vec_docs)
    rb, n_rows, words, qr = _rows(row_bits, qrow)
    n_chunks = -(-n // EXACT_CHUNK)
    ords = begin = ocnt = None
    if ord_lists is not None:
        ocnt = np.array([len(x) for x in ord_lists], np.int32)
        begin = np.concatenate([[0], np.cumsum(ocnt)[:-1]]).astype(np.int64)
        ords = np.ascontiguousarray(np.concatenate([np.asarray(x, np.int32) for x in ord_lists] + [np.zeros(0, np.int32)]), np.int32)
        lists = max(1, -(-int(ocnt.max()) // EXACT_CHUNK))
        n_chunks = max(n_chunks, lists) if (qr[qsel] < 0).any() else lists
    keys = np.zeros((n_sel, n_chunks, k), np.uint64)
    cnt = np.zeros((n_sel, n_chunks), np.int32)
    docs, scores, counts = np.zeros((n_sel, k), np.int32), np.zeros((n_sel, k), np.float32), np.zeros(n_sel, np.int32)
    _check(lib().kh_exact(Q.ctypes.data, nq, D.ctypes.data, n, D.shape[1], sim, qsel.ctypes.data, n_sel, k, n_chunks, _ptr(b),
                          _ptr(f), _ptr(lb), n_docs, _ptr(vd), doc_base, _ptr(rb), n_rows, words, _ptr(qr), _ptr(ords),
                          0 if ords is None else len(ords), _ptr(begin), _ptr(ocnt), keys.ctypes.data, cnt.ctypes.data,
                          docs.ctypes.data, scores.ctypes.data, counts.ctypes.data))
    return keys, cnt, docs, scores, counts


def prepare(D, sim: int):
    """Index-time preparation of a vector field: (norm2 [n], max norm2, ab [n][2])."""
    D = _f32(D)
    n = D.shape[0]
    norm2, mx, ab = np.zeros(n, np.float32), np.zeros(1, np.float32), np.zeros((n, 2), np.float32)
    _check(lib().kh_prepare(D.ctypes.data, n, D.shape[1], sim, norm2.ctypes.data, mx.ctypes.data, ab.ctypes.data))
    return norm2, mx[0], ab


# ---- plain references ----

def key_score(keys) -> np.ndarray:
    """Inverse of make_key's score half."""
    o = (np.asarray(keys, np.uint64) >> np.uint64(32)).astype(np.uint32)
    return np.where(o & 0x80000000, o & 0x7FFFFFFF, ~o).astype(np.uint32).view(np.float32)


def key_ord(keys) -> np.ndarray:
    """Inverse of make_key's ordinal half."""
    return (~np.asarray(keys, np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.int64)


def row_bitmaps(rows) -> np.ndarray:
    """Per-doc 0/1 rows [n_rows][n_docs] -> bitmap rows uint32[n_rows][words]."""
    return np.stack([live_bits(r) for r in rows])


def eligible(ords, n_queries: int, filter_docs=None, live_docs=None, vec_docs=None, rows=None, qrow=None) -> np.ndarray:
    """bool [nq][len(ords)]: the (query, ordinal) pairs a kNN kernel may keep: the ordinal's doc passes the byte filter,
    is live, and is set in the query's row (rows: per-doc 0/1 [n_rows][n_docs]; qrow < 0: no row)."""
    ords = np.asarray(ords, np.int64)
    docs = ords if vec_docs is None else np.asarray(vec_docs, np.int64)[ords]
    ok = np.ones(len(ords), bool)
    if filter_docs is not None:
        ok &= np.asarray(filter_docs)[docs] != 0
    if live_docs is not None:
        ok &= np.asarray(live_docs)[docs] != 0
    out = np.repeat(ok[None, :], n_queries, axis=0)
    for q in range(n_queries):
        if qrow is not None and qrow[q] >= 0:
            out[q] &= np.asarray(rows)[qrow[q]][docs] != 0
    return out


def select_reference(S, kprime: int, chunk_base: int = 0, incoming=None, ok=None) -> list:
    """Per query: the keys of the incoming list and of every eligible entry of S, sorted descending, the first k'."""
    S = _f32(S)
    ords = chunk_base + np.arange(S.shape[1])
    out = []
    for q in range(S.shape[0]):
        m = np.ones(S.shape[1], bool) if ok is None else ok[q]
        keys = make_key(S[q, m], ords[m])
        if incoming is not None:
            keys = np.concatenate([np.asarray(incoming[q], np.uint64), keys])
        out.append(np.sort(keys)[::-1][:kprime])
    return out


SIM_L2, SIM_DOT, SIM_COSINE, SIM_MIP = 0, 1, 2, 3   # NRTGPU_SIM_*


def map_score_reference(sim: int, dims: int, dot, na, nb, d2) -> np.ndarray:
    """VectorSimilarityFunction.compare -> score from float64 sums, in float32 operations (VectorFieldDef.java:664-673;
    byte vectors, sim | BYTE_FLAG, :870-881: DOT_PRODUCT = 0.5 + dot / (dims * 2^15), the rest as for floats)."""
    f = np.float32
    one, two = f(1.0), f(2.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        if sim == (SIM_DOT | BYTE_FLAG):
            return f(0.5) + np.asarray(dot, np.float64).astype(f) / f(dims * (1 << 15))
        base = sim & 0xff
        if base == SIM_L2:
            return one / (one + np.asarray(d2, np.float64).astype(f))
        if base == SIM_MIP:
            t = np.asarray(dot, np.float64).astype(f)
            return np.where(t < 0, one / (one + f(-1.0) * t), t + one).astype(f)
        x = np.asarray(dot, np.float64) if base == SIM_DOT else np.asarray(dot, np.float64) / np.sqrt(np.asarray(na, np.float64) * nb)
        s = (one + x.astype(f)) / two
        return np.where(s > 0, s, f(0.0)).astype(f)   # the cosine of a zero vector is NaN: not > 0, so the score is 0


def exact_scores(Q, D, sim: int, boosts=None) -> np.ndarray:
    """float32 scores [nq][n] of every pair by map_score_reference over float64 sums, x boost in float32."""
    Q, D = np.asarray(Q, np.float64), np.asarray(D, np.float64)
    dot = Q @ D.T
    na, nb = (Q * Q).sum(axis=1)[:, None], (D * D).sum(axis=1)[None, :]
    d2 = np.stack([((D - q[None, :]) ** 2).sum(axis=1) for q in Q])
    s = map_score_reference(sim, Q.shape[1], dot, na, nb, d2)
    if boosts is not None:
        s = s * np.asarray(boosts, np.float32)[:, None]
    return s.astype(np.float32)


def page_reference(scores, k: int, docs=None, ok=None):
    """(docs [k], scores [k], count) of one query: eligible entries by (score desc, doc asc)."""
    scores = np.asarray(scores, np.float32)
    docs = np.arange(len(scores)) if docs is None else np.asarray(docs)
    idx = np.arange(len(scores)) if ok is None else np.nonzero(ok)[0]
    order = idx[np.lexsort((docs[idx], -scores[idx].astype(np.float64)))][:k]
    return docs[order], scores[order], len(order)


def score_upper_bound_reference(sim: int, dims: int, th, qn, dmax, eps, boost) -> float:
    """DESIGN.md 4.3: a vector whose approximate score is <= th has an exact raw score <= th + eps |q| dmax (cosine:
    eps |q| on |q| cos, then divided by |q|; l2: 2 eps |q| dmax on 2 <q, d> - |d|^2); mapped through the monotone score
    mapping, times the boost. float64 throughout."""
    th, qn, dmax, eps, boost = float(th), float(qn), float(dmax), float(eps), float(boost)
    base = sim & 0xff
    if base == SIM_COSINE:
        c = min((th + eps * qn) / qn, 1.0) if qn > 0 else 1.0
        s = max((1.0 + c) / 2.0, 0.0)
    elif base == SIM_L2:
        d2 = max(qn * qn - (th + 2.0 * eps * qn * dmax), 0.0)
        s = 1.0 / (1.0 + d2)
    else:
        x = th + eps * qn * dmax
        if sim == (SIM_DOT | BYTE_FLAG):
            s = max(0.5 + x / (dims * 32768.0), 0.0)
        elif base == SIM_DOT:
            s = max((1.0 + x) / 2.0, 0.0)
        else:
            s = 1.0 / (1.0 - x) if x < 0 else x + 1.0
    return s * boost


def certificate_reference(sim: int, dims: int, th, qn, dmax, eps, boost, kth_score) -> float:
    """Margin of the rank-safety decision: the k-th exact score minus the largest score a vector outside the candidate
    list can have. The query is safe iff the margin is > 0 (strictly)."""
    return float(kth_score) - score_upper_bound_reference(sim, dims, th, qn, dmax, eps, boost)


def approx_unit(sim: int, qn, dmax, eps) -> float:
    """The certificate's error bound in the units of the approximate score."""
    base = sim & 0xff
    return float(eps) * float(qn) * (1.0 if base == SIM_COSINE else 2.0 * float(dmax) if base == SIM_L2 else float(dmax))
